"""CPU: the conv launches of the other benchmarked workloads, through dt_conv_plan (no GPU needed).  test_conv_plan.py
pins the R50-FPN-3D inference step; this file adds the 2-D R50-FPN inference step (`bench.py --config r50fpn2d`), the
R18-3D tube step (`--config r18tube`) and the forward convs of the keypoint R-CNN training step, each at the reduced
shapes tests/test_gpu_conv_workloads.py runs, and the stricter launch key that the coverage test of that file checks."""
import pytest

from test_conv_plan import PLAN_FIELDS, R50_FPN_3D, SMS, conv_args, layer_modes, plan_key, step_plan

# Rows as in test_conv_plan.R50_FPN_3D: (name, N, T, H, W, Cin, Cout, k, stride, pad, res_mode), one per distinct
# dt_conv3d launch of the step.  Layers of one shape but a different fused epilogue (AffineChannel + ReLU of the body,
# bias of the FPN / RPN convs) keep a row each.
P1 = ((1, 1, 1), (1, 1, 1), (0, 0, 0))            # pointwise
S2 = ((1, 1, 1), (1, 2, 2), (0, 0, 0))            # pointwise, stride 2 (folded into the input map)
K33 = ((1, 3, 3), (1, 1, 1), (0, 1, 1))
K333 = ((3, 3, 3), (1, 1, 1), (1, 1, 1))

# 2-D R50-FPN inference: 8 single frames, 800 x 1344 blob (P2 .. P6 = 200x336 .. 13x21), 1000 RoIs per image, 104
# keypoint RoIs per image.  bf16x3 / bf16x3h run the keypoint head's 3x3 convs as Winograd GEMMs (test_gpu_winograd.py):
# those two rows launch dt_conv3d in bf16, tf32 and tf32x3 only.
R50_FPN_2D = [
    ('res2_0 branch1', 8, 1, 200, 336, 64, 256) + P1 + (0,),
    ('res2_0 branch2a', 8, 1, 200, 336, 64, 64) + P1 + (0,),
    ('res2 3x3', 8, 1, 200, 336, 64, 64) + K33 + (0,),
    ('res2 1x1 expand + shortcut', 8, 1, 200, 336, 64, 256) + P1 + (1,),
    ('res2 1x1 reduce', 8, 1, 200, 336, 256, 64) + P1 + (0,),
    ('res3_0 branch1 s2', 8, 1, 200, 336, 256, 512) + S2 + (0,),
    ('res3_0 branch2a s2', 8, 1, 200, 336, 256, 128) + S2 + (0,),
    ('res3 3x3', 8, 1, 100, 168, 128, 128) + K33 + (0,),
    ('res3 expand + shortcut', 8, 1, 100, 168, 128, 512) + P1 + (1,),
    ('res3 1x1 reduce', 8, 1, 100, 168, 512, 128) + P1 + (0,),
    ('res4_0 branch1 s2', 8, 1, 100, 168, 512, 1024) + S2 + (0,),
    ('res4_0 branch2a s2', 8, 1, 100, 168, 512, 256) + S2 + (0,),
    ('res4 3x3', 8, 1, 50, 84, 256, 256) + K33 + (0,),
    ('res4 expand + shortcut', 8, 1, 50, 84, 256, 1024) + P1 + (1,),
    ('res4 1x1 reduce', 8, 1, 50, 84, 1024, 256) + P1 + (0,),
    ('res5_0 branch1 s2', 8, 1, 50, 84, 1024, 2048) + S2 + (0,),
    ('res5_0 branch2a s2', 8, 1, 50, 84, 1024, 512) + S2 + (0,),
    ('res5 3x3', 8, 1, 25, 42, 512, 512) + K33 + (0,),
    ('res5 expand + shortcut', 8, 1, 25, 42, 512, 2048) + P1 + (1,),
    ('res5 1x1 reduce', 8, 1, 25, 42, 2048, 512) + P1 + (0,),
    ('fpn lateral P5', 8, 1, 25, 42, 2048, 256) + P1 + (0,),
    ('fpn lateral P4 + top-down', 8, 1, 50, 84, 1024, 256) + P1 + (2,),
    ('fpn lateral P3 + top-down', 8, 1, 100, 168, 512, 256) + P1 + (2,),
    ('fpn lateral P2 + top-down', 8, 1, 200, 336, 256, 256) + P1 + (2,),
    ('fpn post-hoc P2', 8, 1, 200, 336, 256, 256) + K33 + (0,),
    ('fpn post-hoc P3', 8, 1, 100, 168, 256, 256) + K33 + (0,),
    ('fpn post-hoc P4', 8, 1, 50, 84, 256, 256) + K33 + (0,),
    ('fpn post-hoc P5', 8, 1, 25, 42, 256, 256) + K33 + (0,),
    ('rpn conv P2', 8, 1, 200, 336, 256, 256) + K33 + (0,),
    ('rpn conv P3', 8, 1, 100, 168, 256, 256) + K33 + (0,),
    ('rpn conv P4', 8, 1, 50, 84, 256, 256) + K33 + (0,),
    ('rpn conv P5', 8, 1, 25, 42, 256, 256) + K33 + (0,),
    ('rpn conv P6', 8, 1, 13, 21, 256, 256) + K33 + (0,),
    ('rpn heads P2', 8, 1, 200, 336, 256, 15) + P1 + (0,),
    ('rpn heads P3', 8, 1, 100, 168, 256, 15) + P1 + (0,),
    ('rpn heads P4', 8, 1, 50, 84, 256, 15) + P1 + (0,),
    ('rpn heads P5', 8, 1, 25, 42, 256, 15) + P1 + (0,),
    ('rpn heads P6', 8, 1, 13, 21, 256, 15) + P1 + (0,),
    ('fc6', 1, 1, 1, 8000, 12544, 1024) + P1 + (0,),
    ('fc7', 1, 1, 1, 8000, 1024, 1024) + P1 + (0,),
    ('cls + bbox', 1, 1, 1, 8000, 1024, 10) + P1 + (0,),
    ('keypoint head conv1', 832, 1, 14, 14, 256, 512) + K33 + (0,),
    ('keypoint head conv', 832, 1, 14, 14, 512, 512) + K33 + (0,),
    ('keypoint lowres (sub-pixel deconv)', 832, 1, 14, 14, 512, 68) + K33 + (0,),
]

# R18-3D tube keypoint R-CNN: 8 clips of 3 frames, 800 x 1333 blob (stride-1 blob: the maps are 200x334, 100x167, 50x84).
# Basic blocks whose first 3x3x3 conv strides H and W; a single-level 3-D RPN; the res5 RoI head on 1000 tubes x 3 frames
# of 7 x 7 per clip (ROI_XFORM_RESOLUTION 7: stride_init 1, so res5 keeps 7 x 7); the class / box FC on 8000 x 3 frame
# rows; the 3-D keypoint head on 104 tubes per clip and the per-frame sub-pixel conv.
R18_TUBE = [
    ('res2 3x3', 8, 3, 200, 334, 64, 64) + K33 + (0,),
    ('res2 3x3 + shortcut', 8, 3, 200, 334, 64, 64) + K33 + (1,),
    ('res3_0 branch1 s2', 8, 3, 200, 334, 64, 128) + S2 + (0,),
    ('res3_0 branch2a 3x3x3 s2', 8, 3, 200, 334, 64, 128, (3, 3, 3), (1, 2, 2), (1, 1, 1), 0),
    ('res3 3x3x3 + shortcut', 8, 3, 100, 167, 128, 128) + K333 + (1,),
    ('res3_1 branch2a 3x3x3', 8, 3, 100, 167, 128, 128) + K333 + (0,),
    ('res4_0 branch1 s2', 8, 3, 100, 167, 128, 256) + S2 + (0,),
    ('res4_0 branch2a 3x3x3 s2', 8, 3, 100, 167, 128, 256, (3, 3, 3), (1, 2, 2), (1, 1, 1), 0),
    ('res4 3x3x3 + shortcut', 8, 3, 50, 84, 256, 256) + K333 + (1,),
    ('res4_1 branch2a 3x3x3', 8, 3, 50, 84, 256, 256) + K333 + (0,),
    ('rpn conv 3x3x3', 8, 3, 50, 84, 256, 256) + K333 + (0,),
    ('rpn heads', 8, 3, 50, 84, 256, 60) + P1 + (0,),
    ('res5_0 branch1 (RoI)', 8000, 3, 7, 7, 256, 512) + P1 + (0,),
    ('res5_0 branch2a (RoI)', 8000, 3, 7, 7, 256, 512) + K33 + (0,),
    ('res5 3x3 + shortcut (RoI)', 8000, 3, 7, 7, 512, 512) + K33 + (1,),
    ('res5_1 branch2a (RoI)', 8000, 3, 7, 7, 512, 512) + K33 + (0,),
    ('cls + bbox', 1, 1, 1, 24000, 512, 10) + P1 + (0,),
    ('keypoint head conv1 3x3x3', 832, 3, 14, 14, 256, 512) + K333 + (0,),
    ('keypoint head conv 3x3x3', 832, 3, 14, 14, 512, 512) + K333 + (0,),
    ('keypoint lowres (sub-pixel deconv)', 832, 3, 14, 14, 512, 68) + K33 + (0,),
]

# Forward of KeypointRcnnTrainer.step at the bench training config: 2 clips of 3 frames, 800 x 1344 blob, bf16.  The
# frozen stem and res2 run through the inference engine; res3 .. res5, FPN, RPN and the RoI heads are TrainConv layers
# with the padded output channel counts the trainer packs (RPN 15 -> 16, class / box 10 -> 16, sub-pixel 68 -> 72).
# The FCs run over 2 x 512 sampled RoIs, the keypoint head over 2 x 128 keypoint RoIs.
TRAIN_FWD = [
    ('res2_0 branch1', 2, 3, 200, 336, 64, 256) + P1 + (0,),
    ('res2_0 branch2a', 2, 3, 200, 336, 64, 64) + P1 + (0,),
    ('res2 3x3', 2, 3, 200, 336, 64, 64) + K33 + (0,),
    ('res2 1x1 expand + shortcut', 2, 3, 200, 336, 64, 256) + P1 + (1,),
    ('res2 1x1 reduce', 2, 3, 200, 336, 256, 64) + P1 + (0,),
    ('res3_0 branch1 s2', 2, 3, 200, 336, 256, 512) + S2 + (0,),
    ('res3_0 branch2a s2', 2, 3, 200, 336, 256, 128) + S2 + (0,),
    ('res3 3x3x3', 2, 3, 100, 168, 128, 128) + K333 + (0,),
    ('res3 expand + shortcut', 2, 3, 100, 168, 128, 512) + P1 + (1,),
    ('res3 1x1 reduce', 2, 3, 100, 168, 512, 128) + P1 + (0,),
    ('res4_0 branch1 s2', 2, 3, 100, 168, 512, 1024) + S2 + (0,),
    ('res4_0 branch2a s2', 2, 3, 100, 168, 512, 256) + S2 + (0,),
    ('res4 3x3x3', 2, 3, 50, 84, 256, 256) + K333 + (0,),
    ('res4 expand + shortcut', 2, 3, 50, 84, 256, 1024) + P1 + (1,),
    ('res4 1x1 reduce', 2, 3, 50, 84, 1024, 256) + P1 + (0,),
    ('res5_0 branch1 s2', 2, 3, 50, 84, 1024, 2048) + S2 + (0,),
    ('res5_0 branch2a s2', 2, 3, 50, 84, 1024, 512) + S2 + (0,),
    ('res5 3x3x3', 2, 3, 25, 42, 512, 512) + K333 + (0,),
    ('res5 expand + shortcut', 2, 3, 25, 42, 512, 2048) + P1 + (1,),
    ('res5 1x1 reduce', 2, 3, 25, 42, 2048, 512) + P1 + (0,),
    ('fpn lateral P5', 2, 3, 25, 42, 2048, 256) + P1 + (0,),
    ('fpn lateral P4 + top-down', 2, 3, 50, 84, 1024, 256) + P1 + (2,),
    ('fpn lateral P3 + top-down', 2, 3, 100, 168, 512, 256) + P1 + (2,),
    ('fpn lateral P2 + top-down', 2, 3, 200, 336, 256, 256) + P1 + (2,),
    ('fpn post-hoc P2', 2, 3, 200, 336, 256, 256) + K333 + (0,),
    ('fpn post-hoc P3', 2, 3, 100, 168, 256, 256) + K333 + (0,),
    ('fpn post-hoc P4', 2, 3, 50, 84, 256, 256) + K333 + (0,),
    ('fpn post-hoc P5', 2, 3, 25, 42, 256, 256) + K333 + (0,),
    ('rpn conv P2', 2, 1, 200, 336, 256, 256) + K33 + (0,),
    ('rpn conv P3', 2, 1, 100, 168, 256, 256) + K33 + (0,),
    ('rpn conv P4', 2, 1, 50, 84, 256, 256) + K33 + (0,),
    ('rpn conv P5', 2, 1, 25, 42, 256, 256) + K33 + (0,),
    ('rpn conv P6', 2, 1, 13, 21, 256, 256) + K33 + (0,),
    ('rpn out P2', 2, 1, 200, 336, 256, 16) + P1 + (0,),
    ('rpn out P3', 2, 1, 100, 168, 256, 16) + P1 + (0,),
    ('rpn out P4', 2, 1, 50, 84, 256, 16) + P1 + (0,),
    ('rpn out P5', 2, 1, 25, 42, 256, 16) + P1 + (0,),
    ('rpn out P6', 2, 1, 13, 21, 256, 16) + P1 + (0,),
    ('fc6', 1, 1, 1, 1024, 12544, 1024) + P1 + (0,),
    ('fc7', 1, 1, 1, 1024, 1024, 1024) + P1 + (0,),
    ('cls + bbox', 1, 1, 1, 1024, 1024, 16) + P1 + (0,),
    ('keypoint head conv1', 256, 1, 14, 14, 256, 512) + K33 + (0,),
    ('keypoint head conv', 256, 1, 14, 14, 512, 512) + K33 + (0,),
    ('keypoint lowres (sub-pixel deconv)', 256, 1, 14, 14, 512, 72) + K33 + (0,),
]

# (N, T, H, W) of each row for the value tests, as test_conv_plan.REDUCED: the step's plan and tile, three or more tiles
# per CTA on 132 SMs, a ragged last wave, a partial last tile wherever the step's launch has one, and skipped padding
# taps wherever the step's launch skips any; an even map for the top-down adds.  The smallest such launch in tiles.  Rows whose step launch runs fewer than
# three waves (RPN P6, the FCs of training and of the tube head, the training-size FPN P5) take more images or rows.
REDUCED_2D = {
    'res2_0 branch1': (1, 1, 79, 336),
    'res2_0 branch2a': (1, 1, 148, 336),
    'res2 3x3': (1, 1, 148, 336),
    'res2 1x1 expand + shortcut': (1, 1, 79, 336),
    'res2 1x1 reduce': (1, 1, 148, 336),
    'res3_0 branch1 s2': (1, 1, 145, 336),
    'res3_0 branch2a s2': (4, 1, 145, 336),
    'res3 3x3': (4, 1, 73, 168),
    'res3 expand + shortcut': (1, 1, 73, 168),
    'res3 1x1 reduce': (4, 1, 73, 168),
    'res4_0 branch1 s2': (5, 1, 25, 168),
    'res4_0 branch2a s2': (6, 1, 97, 168),
    'res4 3x3': (6, 1, 49, 84),
    'res4 expand + shortcut': (5, 1, 13, 84),
    'res4 1x1 reduce': (6, 1, 49, 84),
    'res5_0 branch1 s2': (5, 1, 25, 84),
    'res5_0 branch2a s2': (4, 1, 145, 84),
    'res5 3x3': (4, 1, 73, 42),
    'res5 expand + shortcut': (5, 1, 13, 42),
    'res5 1x1 reduce': (4, 1, 73, 42),
    'fpn lateral P5': (5, 1, 118, 42),
    'fpn lateral P4 + top-down': (6, 1, 50, 84),
    'fpn lateral P3 + top-down': (2, 1, 74, 168),
    'fpn lateral P2 + top-down': (1, 1, 80, 336),
    'fpn post-hoc P2': (1, 1, 79, 336),
    'fpn post-hoc P3': (2, 1, 73, 168),
    'fpn post-hoc P4': (6, 1, 49, 84),
    'fpn post-hoc P5': (5, 1, 118, 42),
    'rpn conv P2': (1, 1, 79, 336),
    'rpn conv P3': (2, 1, 73, 168),
    'rpn conv P4': (6, 1, 49, 84),
    'rpn conv P5': (5, 1, 118, 42),
    'rpn conv P6': (32, 1, 37, 21),
    'rpn heads P2': (1, 1, 148, 336),
    'rpn heads P3': (4, 1, 73, 168),
    'rpn heads P4': (4, 1, 148, 84),
    'rpn heads P5': (19, 1, 61, 42),
    'rpn heads P6': (38, 1, 61, 21),
    'fc6': (1, 1, 1, 6273),
    'fc7': (1, 1, 1, 6273),
    'cls + bbox': (1, 1, 1, 50689),
    'keypoint head conv1': (67, 1, 14, 14),
    'keypoint head conv': (67, 1, 14, 14),
    'keypoint lowres (sub-pixel deconv)': (253, 1, 14, 14),
}
REDUCED_TUBE = {
    'res2 3x3': (1, 3, 55, 334),
    'res2 3x3 + shortcut': (1, 3, 55, 334),
    'res3_0 branch1 s2': (1, 3, 199, 334),
    'res3_0 branch2a 3x3x3 s2': (1, 3, 199, 334),
    'res3 3x3x3 + shortcut': (1, 3, 100, 167),
    'res3_1 branch2a 3x3x3': (1, 3, 100, 167),
    'res4_0 branch1 s2': (2, 3, 97, 167),
    'res4_0 branch2a 3x3x3 s2': (2, 3, 97, 167),
    'res4 3x3x3 + shortcut': (2, 3, 49, 84),
    'res4_1 branch2a 3x3x3': (2, 3, 49, 84),
    'rpn conv 3x3x3': (2, 3, 49, 84),
    'rpn heads': (4, 3, 49, 84),
    'res5_0 branch1 (RoI)': (91, 3, 7, 7),
    'res5_0 branch2a (RoI)': (91, 3, 7, 7),
    'res5 3x3 + shortcut (RoI)': (91, 3, 7, 7),
    'res5_1 branch2a (RoI)': (91, 3, 7, 7),
    'cls + bbox': (1, 1, 1, 50689),
    'keypoint head conv1 3x3x3': (23, 3, 14, 14),
    'keypoint head conv 3x3x3': (23, 3, 14, 14),
    'keypoint lowres (sub-pixel deconv)': (85, 3, 14, 14),
}
REDUCED_TRAIN = {
    'res2_0 branch1': (1, 3, 31, 336),
    'res2_0 branch2a': (1, 3, 55, 336),
    'res2 3x3': (1, 3, 55, 336),
    'res2 1x1 expand + shortcut': (1, 3, 31, 336),
    'res2 1x1 reduce': (1, 3, 55, 336),
    'res3_0 branch1 s2': (1, 3, 51, 336),
    'res3_0 branch2a s2': (1, 3, 199, 336),
    'res3 3x3x3': (1, 3, 100, 168),
    'res3 expand + shortcut': (1, 3, 26, 168),
    'res3 1x1 reduce': (1, 3, 100, 168),
    'res4_0 branch1 s2': (1, 3, 51, 168),
    'res4_0 branch2a s2': (2, 3, 97, 168),
    'res4 3x3x3': (2, 3, 49, 84),
    'res4 expand + shortcut': (1, 3, 26, 84),
    'res4 1x1 reduce': (2, 3, 49, 84),
    'res5_0 branch1 s2': (1, 3, 49, 84),
    'res5_0 branch2a s2': (4, 3, 49, 84),
    'res5 3x3x3': (4, 3, 25, 42),
    'res5 expand + shortcut': (1, 3, 25, 42),
    'res5 1x1 reduce': (4, 3, 25, 42),
    'fpn lateral P5': (5, 3, 40, 42),
    'fpn lateral P4 + top-down': (2, 3, 50, 84),
    'fpn lateral P3 + top-down': (1, 3, 50, 168),
    'fpn lateral P2 + top-down': (1, 3, 32, 336),
    'fpn post-hoc P2': (1, 3, 31, 336),
    'fpn post-hoc P3': (1, 3, 49, 168),
    'fpn post-hoc P4': (2, 3, 49, 84),
    'fpn post-hoc P5': (5, 3, 40, 42),
    'rpn conv P2': (1, 1, 79, 336),
    'rpn conv P3': (2, 1, 73, 168),
    'rpn conv P4': (2, 1, 148, 84),
    'rpn conv P5': (5, 1, 118, 42),
    'rpn conv P6': (32, 1, 37, 21),
    'rpn out P2': (1, 1, 148, 336),
    'rpn out P3': (2, 1, 148, 168),
    'rpn out P4': (4, 1, 148, 84),
    'rpn out P5': (19, 1, 61, 42),
    'rpn out P6': (38, 1, 61, 21),
    'fc6': (1, 1, 1, 6273),
    'fc7': (1, 1, 1, 6273),
    'cls + bbox': (1, 1, 1, 50689),
    'keypoint head conv1': (67, 1, 14, 14),
    'keypoint head conv': (67, 1, 14, 14),
    'keypoint lowres (sub-pixel deconv)': (253, 1, 14, 14),
}


# A strided 3x3 conv on stacks of 32 small maps: the strided activation box over stacked images, with the live taps of
# each tile under stride and a ragged last stack.  No benchmarked launch takes this path today (the tube head's res5
# runs unstrided at ROI_XFORM_RESOLUTION 7); it is what res5_0 branch2a becomes on 7 x 7 RoI maps with stride 2.
STACKED_STRIDED = ('res5_0 branch2a s2 on 7x7 RoI maps', 8000, 3, 7, 7, 256, 512, (1, 3, 3), (1, 2, 2), (0, 1, 1), 0)
STACKED_STRIDED_REDUCED = {STACKED_STRIDED[0]: (283, 3, 7, 7)}


def modes_2d(layer):
    """bf16, tf32, tf32x3, bf16x3 (+ f16 for the post-hoc FPN convs of bf16x3h); the keypoint head's 3x3 convs are
    Winograd GEMMs in the bf16x3 modes."""
    if layer[0].startswith('keypoint head'):
        return ('bf16', 'tf32', 'tf32x3')
    return layer_modes(layer)


def modes_tube(layer):
    """bf16x3h is bf16x3 on the tube graph (no post-hoc FPN convs)."""
    return ('bf16', 'tf32', 'tf32x3', 'bf16x3')


def modes_train(layer):
    return ('bf16',)


# workload -> (rows, reduced shapes, engine modes of a row)
TABLES = {
    'r50fpn2d': (R50_FPN_2D, REDUCED_2D, modes_2d),
    'r18tube': (R18_TUBE, REDUCED_TUBE, modes_tube),
    'train': (TRAIN_FWD, REDUCED_TRAIN, modes_train),
}
CASES = [(wl, l, m) for wl, (rows, _, modes) in TABLES.items() for l in rows for m in modes(l)]


def row_plan(wl, layer, mode, reduced=False):
    return step_plan(layer, mode, reduced, shapes=TABLES[wl][1])


def out_shape(layer, shape=None):
    """(N, To, Ho, Wo) of a row, at its step shape or at `shape` = (N, T, H, W)."""
    N, T, H, W = shape or layer[1:5]
    k, s, p = layer[7:10]
    return N, (T + 2 * p[0] - k[0]) // s[0] + 1, (H + 2 * p[1] - k[1]) // s[1] + 1, (W + 2 * p[2] - k[2]) // s[2] + 1


def ragged_axes(layer, o, shape=None):
    """The axes along which the launch's last tile is partial: image stack, frames, rows, columns."""
    N, To, Ho, Wo = out_shape(layer, shape)
    return {a for a, n, t in (('N', N, o.TB), ('T', To, o.TT), ('H', Ho, o.TH), ('W', Wo, o.TW)) if n % t}


def skips_taps(o):
    """Some tile issues fewer than all its (tap, channel chunk) groups: a tap's activation box lies wholly in the zero
    padding (the kernel's tile_live).  dt_conv_plan counts the MMA k-blocks the launch issues."""
    return o.mma_kblocks < o.kiters * o.tiles


def plan_key_v2(dtype, x3, out_f32, res_mode, o, k, s):
    """plan_key plus what else selects the kernel's address arithmetic: the filter taps, the stride (TMA element strides
    of the activation box, live-tap ranges under stride), image / frame stacking in the M tile, and the residual path
    (TMA ring or per-thread loads)."""
    res = 'tma' if o.nrbuf > 0 else ('ldg' if res_mode else 'none')
    return plan_key(dtype, x3, out_f32, res_mode, o) + (tuple(k), tuple(s), o.TB > 1, o.TT > 1, res)


def row_key(layer, mode, o, v2=True):
    a = conv_args(layer, mode)
    if not v2:
        return plan_key(a['dtype'], a['x3'], a['out_f32'], layer[10], o)
    return plan_key_v2(a['dtype'], a['x3'], a['out_f32'], layer[10], o, layer[7], layer[8])


def table_keys(wl, v2=True):
    """{plan key: [(row name, mode)]} of a workload's step ('r50fpn3d': test_conv_plan.R50_FPN_3D)."""
    rows, _, modes = TABLES[wl] if wl != 'r50fpn3d' else (R50_FPN_3D, None, layer_modes)
    keys = {}
    for l in rows:
        for m in modes(l):
            keys.setdefault(row_key(l, m, step_plan(l, m), v2), []).append((l[0], m))
    return keys


@pytest.mark.parametrize('wl,layer,mode', CASES, ids=['%s-%s-%s' % (w, l[0], m) for w, l, m in CASES])
def test_workload_row_plan_fits(wl, layer, mode):
    o = row_plan(wl, layer, mode)
    assert o.TB * o.TT * o.TH * o.TW <= 128 and o.tiles >= 1
    assert o.stages >= 2 and o.ks in (1, 2) and o.BN in (32, 64, 128)
    assert o.ncbuf in (1, 2, 4) and o.nrbuf in (0, 1, 2, 4)


@pytest.mark.parametrize('wl,layer,mode', CASES, ids=['%s-%s-%s' % (w, l[0], m) for w, l, m in CASES])
def test_reduced_shape_keeps_the_step_plan_over_three_waves(wl, layer, mode):
    """The value tests of test_gpu_conv_workloads.py run each row at its reduced shape.  That launch must take the step's
    plan and M tile, at least three tiles per CTA with a ragged last wave, a
    partial last tile along every axis the step's launch has one on, and skipped padding taps if the step's launch skips
    any (a strided box, a stacked or a ragged tile is where the kernel's coordinates can go wrong)."""
    full, red = row_plan(wl, layer, mode), row_plan(wl, layer, mode, reduced=True)
    shape = TABLES[wl][1][layer[0]]
    for f in PLAN_FIELDS:
        assert getattr(red, f) == getattr(full, f), (f, getattr(red, f), getattr(full, f))
    assert (red.TB, red.TT, red.TH, red.TW) == (full.TB, full.TT, full.TH, full.TW)
    if layer[10] == 2:                     # the top-down add needs an even map; even tile: the coarser map's TMA box
        assert out_shape(layer, shape)[2] % 2 == 0 and out_shape(layer, shape)[3] % 2 == 0
        assert (red.TH % 2, red.TW % 2) == (full.TH % 2, full.TW % 2)
    assert (red.TT > 1, red.TB > 1) == (full.TT > 1, full.TB > 1)
    assert red.tiles >= 3 * SMS and red.tiles % SMS != 0, red.tiles
    assert ragged_axes(layer, full) <= ragged_axes(layer, red, shape), (ragged_axes(layer, full), ragged_axes(layer, red, shape))
    assert skips_taps(red) or not skips_taps(full)
    assert row_key(layer, mode, red) == row_key(layer, mode, full)


@pytest.mark.parametrize('wl', sorted(TABLES))
def test_step_rows_shrink_unless_the_step_runs_under_three_waves(wl):
    """A reduced shape is no larger than the step's along any axis, except where the step's launch runs fewer than three
    waves: there it takes more images or rows instead (the coarsest RPN level, the few-row FCs of training)."""
    rows, shapes, modes = TABLES[wl]
    assert set(shapes) == {l[0] for l in rows}
    for l in rows:
        grown = any(a > b for a, b in zip(shapes[l[0]], l[1:5]))
        if grown:
            assert row_plan(wl, l, modes(l)[0]).tiles < 3 * SMS, l[0]


def test_old_key_collides_across_stride_and_stacking():
    """The plan key of test_conv_plan (storage, residual kind and schedule) cannot tell a strided launch from an
    unstrided one, or stacked images from one image: an R18 tube launch no value test ran matched an R50-FPN-3D row on
    it.  plan_key_v2 keeps such launches apart."""
    old = {}
    for wl in ('r50fpn3d',) + tuple(TABLES):
        rows, _, modes = TABLES[wl] if wl != 'r50fpn3d' else (R50_FPN_3D, None, layer_modes)
        for l in rows:
            for m in modes(l):
                o = step_plan(l, m)
                old.setdefault(row_key(l, m, o, v2=False), set()).add((row_key(l, m, o), wl, l[0], m))
    collide = [v for v in old.values() if len({k[-4:-1] for k, _, _, _ in v}) > 1]
    assert collide
    # the strided 3x3x3 branch2a of R18 res4_0 shares its old key with an unstrided R50-FPN-3D row
    tube = next(v for v in collide for _, wl, name, m in v if (wl, name, m) == ('r18tube', 'res4_0 branch2a 3x3x3 s2', 'bf16'))
    assert any(wl == 'r50fpn3d' and k[-4] == (1, 1, 1) for k, wl, _, _ in tube), tube


def test_plan_key_v2_counts(record_property):
    """The number of distinct launch keys per workload (reported; each is a row of a value-tested table)."""
    for wl in ('r50fpn3d',) + tuple(TABLES):
        n = len(table_keys(wl))
        record_property('plan_keys_v2_' + wl, n)
        assert n >= len(table_keys(wl, v2=False))


@pytest.mark.parametrize('mode', ('bf16', 'tf32', 'tf32x3', 'bf16x3'))
def test_stacked_strided_case_keeps_32_image_stacks(mode):
    """The reduced strided RoI conv keeps the step-size launch's plan and its 32-image stacks of one output row of four
    columns, with 27 images in the last stack and padding taps skipped."""
    full = step_plan(STACKED_STRIDED, mode)
    red = step_plan(STACKED_STRIDED, mode, True, STACKED_STRIDED_REDUCED)
    assert (full.TB, full.TT, full.TH, full.TW) == (red.TB, red.TT, red.TH, red.TW) == (32, 1, 1, 4)
    assert all(getattr(red, f) == getattr(full, f) for f in PLAN_FIELDS)
    assert ragged_axes(STACKED_STRIDED, red, STACKED_STRIDED_REDUCED[STACKED_STRIDED[0]]) == {'N'}
    assert skips_taps(red) and skips_taps(full)
    assert red.tiles >= 3 * SMS and red.tiles % SMS != 0

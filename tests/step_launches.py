"""Library calls of the benchmarked steps, recorded once per pytest process for the launch-table coverage tests
(test_gpu_box_step, test_gpu_dense_step, test_gpu_conv_workloads, test_gpu_train_step_ops, test_gpu_train_grads,
test_gpu_soft_nms, test_gpu_winograd).  Each test keeps its own table and launch key and reads them off record(run).

Runs, built as bench.py builds them:
  (workload, mode)  DetectionEngine construction and detect of one 800 x 1333 clip (not taken where the engine raises
                    NotImplementedError);
  'train'           KeypointRcnnTrainer construction and step as `bench.py --train` runs it;
  'augment'         then, on that trainer, a step_clips of an 800 x 1333 clip at scale 800 and a mirrored 720 x 1280 clip
                    drawn to 640 (TRAIN.AUGMENT);
  'trunk'           RpnTrainer construction and step as `bench.py --train-trunk` runs it.
A run executes on the first record() that asks for it.  Its calls are (name, args, in_backward): args copied at call time,
so a key computed afterwards sees what was passed even where the caller reuses a struct; in_backward is true inside
TrainConv.backward.  A record keeps no device tensor."""
import collections
import ctypes as C

WORKLOADS = ('r50fpn3d', 'r50fpn2d', 'r18tube')
MODES = ('bf16', 'tf32', 'tf32x3', 'bf16x3', 'bf16x3h')
ENGINE_RUNS = tuple((wl, mode) for wl in WORKLOADS for mode in MODES)
CONV_WRAPPERS = ('conv3d', 'conv1_7x7s2', 'conv1_7x7s2_f32')

# conv_py: Python-level calls of the CONV_WRAPPERS of ops/conv.py; facts: what the coverage tests read off the live model
Record = collections.namedtuple('Record', 'taken calls conv_py facts')
_records = {}


def record(run):
    """The Record of `run` (a tag of the module docstring), executing the run if no test has asked for it yet."""
    if run not in _records:
        try:
            _records.update(_trainer(run) if run in ('train', 'augment', 'trunk') else {run: _engine(*run)})
        finally:
            from test_gpu_engine import _cfg
            _cfg()
    return _records[run]


def conv_plan(a):
    """(descriptor, dt_conv_plan) of a recorded dt_conv3d call's arguments."""
    from detectandtrack_b200 import _lib as L
    d, o = a[0]._obj, L.ConvPlan()
    aligned = a[5] is None or a[5].value % 16 == 0
    assert L.lib().dt_conv_plan(C.byref(d), int(aligned), C.byref(o)) == 0, L.lib().dt_last_error()
    return d, o


def _snapshot(a):
    """One L.call argument as it is now: ctypes values, structs and arrays copied, byref of a copy, others as they are."""
    if isinstance(a, (C.Structure, C.Union, C.Array, C._SimpleCData)):
        return type(a).from_buffer_copy(a)
    if type(a).__name__ == 'CArgObject':                # C.byref(x)
        return C.byref(_snapshot(a._obj))
    return a


def _recorded(body):
    """Run body() with every L.call recorded; body returns its facts dict, or None when the run is not taken."""
    import torch
    from detectandtrack_b200 import _lib as L
    from detectandtrack_b200.modeling.trainer import TrainConv
    from detectandtrack_b200.ops import conv as cv
    calls, n = [], dict(py=0, bwd=0)
    call, backward, wrapped = L.call, TrainConv.backward, {f: getattr(cv, f) for f in CONV_WRAPPERS}

    def spy(name, *a):
        calls.append((name, tuple(_snapshot(x) for x in a), n['bwd'] > 0))
        return call(name, *a)

    def counted(f):
        def conv(*a, **kw):
            n['py'] += 1
            return f(*a, **kw)
        return conv

    def in_backward(self, *a, **kw):
        n['bwd'] += 1
        try:
            return backward(self, *a, **kw)
        finally:
            n['bwd'] -= 1
    L.call, TrainConv.backward = spy, in_backward
    for f, fn in wrapped.items():
        setattr(cv, f, counted(fn))
    try:
        facts = body()
        torch.cuda.synchronize()
    finally:
        L.call, TrainConv.backward = call, backward
        for f, fn in wrapped.items():
            setattr(cv, f, fn)
    return Record(facts is not None, calls, n['py'], facts or {})


def _engine(wl, mode):
    import torch
    import bench
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling.engine import DetectionEngine
    cfg = bench.bench_cfg(800, 1333, wl)
    blobs, spec = P.random_blobs(cfg)
    frames = torch.from_numpy(bench.synth_frames(1, bench.frames_per_clip(cfg), 800, 1333, 7)).cuda()

    def run():
        try:
            eng = DetectionEngine(cfg, blobs, spec, dtype=mode)
        except NotImplementedError:
            return None
        eng.detect(frames)
        return dict(wino_kps=eng.wino_kps, kps_convs=len(eng.kps_convs))
    return _recorded(run)


def _trainer(run):
    """{'trunk': Record} or {'train': Record, 'augment': Record} (one trainer)."""
    import numpy as np
    import torch
    import bench
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling.trainer import KeypointRcnnTrainer, RpnTrainer, pack_gt
    cfg = bench.bench_cfg(800, 1333, 'r50fpn3d')
    cfg.TRAIN.BATCH_SIZE_PER_IM = 512; cfg.TRAIN.RPN_PRE_NMS_TOP_N = 2000
    blobs, spec = P.random_blobs(cfg)
    frames = torch.from_numpy(bench.synth_frames(2, 3, 800, 1333, 100)).cuda()
    tr = []

    def trunk():
        rt = RpnTrainer(cfg, blobs, spec)
        rt.step(frames, rt.synthetic_targets(2, 800, 1333, seed=0))
        return {}

    def step():
        tr.append(KeypointRcnnTrainer(cfg, blobs, spec))
        tr[0].step(frames, pack_gt(bench.synth_gt(2, 800, 1333, 7)))
        return _train_facts(tr[0])

    def augment():
        rng = np.random.RandomState(3)
        clips = [torch.from_numpy(rng.randint(0, 256, (3, h, w, 3)).astype(np.uint8)).cuda() for h, w in ((800, 1333), (720, 1280))]
        gt = pack_gt(bench.synth_gt(1, 800, 1333, 3) + bench.synth_gt(1, 720, 1280, 4))
        tr[0].step_clips(clips, gt, [800, 640], [0, 1], seed=5)
        return {}
    if run == 'trunk':
        return dict(trunk=_recorded(trunk))
    return dict(train=_recorded(step), augment=_recorded(augment))


def _train_facts(tr):
    """The trainer's conv count, and after the update the nonzero entries of what must stay zero in the master, forward
    and dgrad filters: per padded output conv (its padding filter rows, those entries, its padding biases), and the
    sub-pixel deconv's dead taps (their count, those entries)."""
    import torch
    padding = {}
    for name, c, live in (('rpn_out', tr.rpn_out, 5 * tr.A), ('cls_bbox', tr.cls_bbox, 5 * tr.C_), ('kps_lowres', tr.kps_lowres, 4 * tr.K)):
        nz = int((c.w[:, live:] != 0).sum() + (c.w_fwd[:, live:] != 0).sum() + (c.w_dg[:, :, live:] != 0).sum())
        padding[name] = (c.cout - live, nz, int((c.bias[live:] != 0).sum()))
    K, kl = tr.K, tr.kps_lowres
    dead = torch.ones((9, kl.cout), dtype=torch.bool)
    for sub in range(4):
        for tap in range(9):
            if 0 <= (sub >> 1) + 3 - 2 * (tap // 3) <= 3 and 0 <= (sub & 1) + 3 - 2 * (tap % 3) <= 3:
                dead[tap, sub * K:(sub + 1) * K] = False
    dead = dead.cuda()
    nz = int((kl.w[dead] != 0).sum() + (kl.w_fwd[dead] != 0).sum() + (kl.w_dg.flip(0).permute(0, 2, 1)[dead] != 0).sum())
    return dict(convs=len(tr.convs), padding=padding, dead_taps=(int(dead.sum()), nz))

"""CPU: the frozen-backbone training step's host logic.  The all-reduce schedule of a backward pass that produces only the head's gradients
(nerf_rpn_b200.train.bucket_schedule with a lower bound), and the reference's unmodified driver with --freeze_backbone building a model whose
training forward takes the frozen-backbone step (run_rpn.py:193-195)."""
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "nerf_rpn")


def _config4_bucket():
    """(offsets the full backward pass finalises, in construction order, head offset, parameter count) of ResNet50-FPN + anchor head (--rotated_bbox)."""
    from nerf_rpn_b200.model.anchor import RPNHead
    from nerf_rpn_b200.model.feature_extractor import Bottleneck, ResNet_FPN_256
    bb = ResNet_FPN_256(Bottleneck, [3, 4, 6, 3], input_dim=4, is_max_pool=True)
    head = RPNHead(256, 13, 4, rotate=True)
    params = list(bb.parameters()) + list(head.parameters())
    off, o = {}, 0
    for p in params:
        off[id(p)] = o
        o += p.numel()
    n = o
    head_lo = n - sum(p.numel() for p in head.parameters())
    blocks = [blk for stage in bb.layers for blk in stage]
    bwd_lo = [0] + [off[id(blk.conv1.weight)] for blk in blocks] + [min(off[id(m.weight)] for m in list(bb.latlayers) + list(bb.smooths)), head_lo]
    return bwd_lo, head_lo, n


def _covers_once(sched, lo, hi):
    ranges = [(a, b) for _, a, b in sched]
    assert [k for k, _, _ in sched] == sorted(k for k, _, _ in sched)                 # launch order
    assert ranges == sorted(ranges, reverse=True)                                     # from the end of the bucket towards its start
    assert ranges[0][1] == hi and ranges[-1][0] == lo
    assert all(ranges[i][0] == ranges[i + 1][1] for i in range(len(ranges) - 1))       # disjoint and contiguous


@pytest.mark.parametrize("bucket_mb", [1.0, 16.0, 32.0, 1024.0])
def test_bucket_schedule_covers_head_range_once(bucket_mb):
    from nerf_rpn_b200.train import bucket_schedule
    _, head_lo, n = _config4_bucket()
    bucket = int(bucket_mb * (1 << 20) / 4)
    assert (bucket < n - head_lo) == (bucket_mb <= 16.0)                                # bucket sizes on both sides of the head's 7.1 M elements
    assert bucket_schedule([head_lo], n, bucket) == ([] if bucket > n - head_lo else [(0, head_lo, n)])   # without a lower bound: as before
    sched = bucket_schedule([head_lo], n, bucket, lowest=head_lo)
    assert sched == [(0, head_lo, n)]
    _covers_once(sched, head_lo, n)


@pytest.mark.parametrize("bucket_mb", [1.0, 8.0, 32.0, 1024.0])
def test_bucket_schedule_default_unchanged(bucket_mb):
    """The full backward pass: the default lower bound 0 gives the schedule of an explicit lowest=0, covering the whole bucket."""
    from nerf_rpn_b200.train import bucket_schedule
    bwd_lo, _, n = _config4_bucket()
    bucket = int(bucket_mb * (1 << 20) / 4)
    sched = bucket_schedule(bwd_lo, n, bucket)
    assert sched == bucket_schedule(bwd_lo, n, bucket, lowest=0)
    _covers_once(sched, 0, n)
    assert bucket_schedule([0, 5, 9, 20], 30, 4) == [(0, 20, 30), (1, 9, 20), (2, 5, 9), (3, 0, 5)]
    assert bucket_schedule([0, 5, 9, 20], 30, 12) == [(1, 9, 30), (3, 0, 9)]


@pytest.mark.skipif(not os.path.isdir(REF), reason="oracle/_ref not staged")
def test_reference_driver_freeze_backbone_selects_frozen_step(tmp_path):
    code = textwrap.dedent(f"""
        import sys, types
        sys.path[:0] = [{os.path.join(ROOT, 'dropin')!r}, {ROOT!r}, {REF!r}]
        sys.modules['wandb'] = types.ModuleType('wandb')
        import model
        import numpy as np, pandas as pd, torch
        np.savez('{tmp_path}/s.npz', rgbsigma=np.random.rand(32, 32, 32, 4).astype('float32'))
        np.save('{tmp_path}/s.npy', np.array([[2, 2, 2, 9, 9, 9, 0.1]], dtype='float32'))
        pd.DataFrame(dict(scene=['s'], rgbsigma_path=['{tmp_path}/s.npz'], boxes_path=['{tmp_path}/s.npy'])).to_csv('{tmp_path}/t.csv')
        base = ['run_rpn.py', '--mode', 'eval', '--dataset_name', 'general', '--test_csv', '{tmp_path}/t.csv', '--backbone_type', 'resnet',
                '--resolution', '32', '--rotated_bbox']
        import run_rpn                                                   # the reference's unmodified driver
        sys.argv = base + ['--freeze_backbone']
        tr = run_rpn.Trainer(run_rpn.parse_args())
        m = tr.model
        assert type(m).__module__.startswith('nerf_rpn_b200.'), type(m).__module__
        assert not any(p.requires_grad for p in m.backbone.parameters())
        assert all(p.requires_grad for p in m.rpn.head.parameters())
        assert m.frozen_backbone()
        sys.argv = base
        assert not run_rpn.Trainer(run_rpn.parse_args()).model.frozen_backbone()
        m.backbone.latlayers[0].weight.requires_grad_(True)             # a partial pattern keeps the full step
        assert not m.frozen_backbone()
        print('OK')
    """)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                       env={**os.environ, "CUDA_VISIBLE_DEVICES": "", "WANDB_MODE": "disabled"})
    assert r.returncode == 0, r.stderr[-3000:]
    assert "OK" in r.stdout

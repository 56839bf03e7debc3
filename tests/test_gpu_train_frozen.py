"""GPU: the frozen-backbone training step (run_rpn.py --freeze_backbone: every ResNet_FPN_256 parameter has requires_grad = False, BatchNorm
still in train mode).  The engine runs only the head's backward, and clip, AdamW and the all-reduce cover the head's range of the flat buffers.
Checked against the full step of the same engine (same kernels in the same order: bit for bit), against the unmodified reference in train mode
with its backbone frozen, and through the drop-in loop of run_rpn.py:384-395."""
import pytest
import torch

from tests.test_gpu_train import _grad_metrics, _planted
from tests.test_gpu_train_ragged import _model, _need_ref

pytestmark = pytest.mark.gpu

DIMS = (64, 96, 80)


def _engine(layers, rotated, precision, frozen, **kw):
    from nerf_rpn_b200.train import RPNTrainEngine
    return RPNTrainEngine(_model(layers, rotated), precision=precision, seed=7, freeze_backbone=frozen, **kw)


# ------------------------------------------------------------------------------------------------ 1. bit identity with the full step
@pytest.mark.parametrize("layers", [(2, 1, 1, 1), (3, 4, 6, 3)])
@pytest.mark.parametrize("rotated,precision", [(True, "bf16"), (False, "bf16"), (True, "fp16"), (False, "fp16")])
def test_frozen_step_bit_identical_to_full_step_head(layers, rotated, precision):
    """Same seed-0 weights, input, targets and sampler seed: losses and the head's gradients (the tail of flat_g) of the frozen step equal
    the full step's bit for bit, in the two eager runs and the captured-graph replays that follow; the backbone's gradients stay untouched."""
    grid, gt = _planted(DIMS, 12, 11, rotated)
    grid, gt = grid.cuda()[None], [gt.cuda()]
    full, frozen = _engine(layers, rotated, precision, False), _engine(layers, rotated, precision, True)
    assert full.head_lo == frozen.head_lo
    lo = full.head_lo
    for it in range(4):                                          # eager, eager, capture + replay, replay
        lf = full.forward_backward(grid, gt).clone()
        lz = frozen.forward_backward(grid, gt).clone()
        torch.cuda.synchronize()
        assert torch.equal(lf, lz), (it, lf.tolist(), lz.tolist())
        assert torch.equal(full.flat_g[lo:], frozen.flat_g[lo:]), it
        assert not frozen.flat_g[:lo].any()
    plan = frozen.plan(1, DIMS)
    assert len(plan.bwd) == 1 and plan.bwd_lo == [lo]
    assert frozen.cache_stats()["graphs"] == 2                   # the forward and the (shorter) backward list replay as CUDA graphs


# ------------------------------------------------------------------------------------------------ 2. against the reference
def _reference_frozen_step(ref_gpu, rotated, layers, grid, gt, autocast_dtype=None):
    """The unmodified reference in train mode with every backbone parameter frozen (run_rpn.py:193-195)."""
    m = ref_gpu.build_reference_model(rotated=rotated, seed=0, layers=layers, rpn_fg_iou_thresh=0.35, rpn_bg_iou_thresh=0.2).cuda().train()
    for p in m.backbone.parameters():
        p.requires_grad = False
    out = dict(bsd={k: v.detach().clone() for k, v in m.backbone.state_dict().items()}, hsd={k: v.detach().clone() for k, v in m.rpn.head.state_dict().items()})
    rec = {}
    orig = m.rpn.fg_bg_sampler

    def recording_sampler(labels):
        pos, neg = orig(labels)
        rec["pos"] = [torch.where(m_)[0] for m_ in pos]; rec["neg"] = [torch.where(m_)[0] for m_ in neg]
        return pos, neg
    m.rpn.fg_bg_sampler = recording_sampler
    torch.manual_seed(123)
    ctx = torch.autocast("cuda", dtype=autocast_dtype) if autocast_dtype is not None else torch.autocast("cuda", enabled=False)
    with ctx:
        _, losses, _ = m([grid], [gt])
        loss = losses["loss_objectness"] + 5.0 * losses["loss_rpn_box_reg"]
    loss.backward()
    assert all(p.grad is None for p in m.backbone.parameters())
    out["names"] = ["head." + n for n, _ in m.rpn.head.named_parameters()]
    out["grads"] = [p.grad.detach().float().clone() for p in m.rpn.head.parameters()]
    out["losses"] = (losses["loss_objectness"].item(), losses["loss_rpn_box_reg"].item())
    out["samples"] = (rec["pos"][0], rec["neg"][0])
    out["running"] = {k: v.detach().float().clone() for k, v in m.backbone.state_dict().items() if "running" in k}
    del m
    torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize("layers,rotated,precision", [((2, 1, 1, 1), True, "fp16"), ((3, 4, 6, 3), False, "bf16")])
def test_frozen_step_vs_reference_with_frozen_backbone(layers, rotated, precision):
    """Losses and head gradients against the reference's fp32 autograd, held to its own autocast run like the full step is
    (tests/test_gpu_train.py::_training_step_parity); the backbone's BatchNorm running statistics after the step by the same per-tensor rule;
    and on the drop-in path no backbone parameter receives a gradient."""
    ref_gpu = _need_ref()
    grid, gt = _planted(DIMS, 12, 11, rotated)
    grid, gt = grid.cuda(), gt.cuda()
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
    try:
        r32 = _reference_frozen_step(ref_gpu, rotated, layers, grid, gt)
        rac = _reference_frozen_step(ref_gpu, rotated, layers, grid, gt, torch.bfloat16 if precision == "bf16" else torch.float16)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    from nerf_rpn_b200.train import RPNTrainEngine
    model = _model(layers, rotated, ref_state=r32)
    for p in model.backbone.parameters():
        p.requires_grad = False
    eng = RPNTrainEngine(model, precision=precision, reg_loss_weight=5.0, freeze_backbone=True)
    plan = eng.plan(1, DIMS)
    torch.manual_seed(123)
    got_l = eng.forward_backward(grid[None], [gt]).tolist()
    torch.cuda.synchronize()
    pos_o, neg_o, _ = plan.last_samples[0]
    same = set(pos_o.tolist()) == set(r32["samples"][0].tolist()) and set(neg_o.tolist()) == set(r32["samples"][1].tolist())
    inv = 1.0 / eng.loss_scale
    grads = [eng.grad_of(p).view(p.shape).clone() * inv for p in model.rpn.head.parameters()]
    cos_o, rel_o, per_o = _grad_metrics(grads, r32)
    cos_a, rel_a, per_a = _grad_metrics(rac["grads"], r32)
    running = {k: v.float() for k, v in model.backbone.state_dict().items() if "running" in k}

    def rel(a, b):
        return ((a - b).norm() / (b.norm() + 1e-30)).item()
    bn_o = {k: rel(running[k], r32["running"][k]) for k in running}
    bn_a = {k: rel(rac["running"][k], r32["running"][k]) for k in running}
    tag = f"[{layers} {'OBB' if rotated else 'AABB'} {precision} frozen backbone]"
    print(f"{tag} losses: ours {got_l}  reference fp32 {r32['losses']}  reference autocast {rac['losses']}")
    print(f"{tag} head gradient vs reference fp32: ours cosine {cos_o:.4f} rel {rel_o:.3f} | reference autocast cosine {cos_a:.4f} rel {rel_a:.3f}")
    print(f"{tag} running statistics, worst rel err: ours {max(bn_o.values()):.3e} autocast {max(bn_a.values()):.3e}")
    checks = [(same, "the sampler did not reproduce the reference's draws")]
    for k in range(2):
        e_o, e_a = abs(got_l[k] - r32["losses"][k]), abs(rac["losses"][k] - r32["losses"][k])
        slack = (1e-2 if precision == "bf16" else 3e-3) * abs(r32["losses"][k])
        checks.append((e_o <= 3.0 * e_a + slack, f"loss {k}: ours off by {e_o}, autocast by {e_a}"))
    checks.append((cos_o >= cos_a - 0.08, f"gradient cosine {cos_o} vs autocast {cos_a}"))
    checks.append((rel_o <= 1.15 * rel_a + 0.02, f"gradient rel err {rel_o} vs autocast {rel_a}"))
    bad = [(n, v, per_a[n]) for n, v in per_o.items() if v > 1.25 * per_a[n] + 0.03]
    checks.append((not bad, f"tensors worse than the autocast reference: {bad[:5]}"))
    bad_bn = [(k, bn_o[k], bn_a[k]) for k in bn_o if bn_o[k] > 1.25 * bn_a[k] + 0.03]
    checks.append((not bad_bn, f"running statistics worse than the autocast reference: {bad_bn[:5]}"))
    changed = [k for k in running if not torch.equal(running[k], r32["bsd"][k].float())]
    checks.append((len(changed) == len(running), "BatchNorm running statistics were not updated"))
    failed = [msg for ok, msg in checks if not ok]
    assert not failed, failed
    # the drop-in path: autograd hands gradients to the head only
    model._train_engine = None
    torch.manual_seed(123)
    _, losses, _ = model([grid], [gt])
    (losses["loss_objectness"] + 5.0 * losses["loss_rpn_box_reg"]).backward()
    assert all(p.grad is None for p in model.backbone.parameters())
    assert all(p.grad is not None for p in model.rpn.head.parameters())


# ------------------------------------------------------------------------------------------------ 3. optimizer
@pytest.mark.parametrize("precision", ["bf16", "fp16"])
def test_frozen_optimizer_step_updates_head_only(precision):
    """Several train_steps: the backbone's master weights and AdamW moments are bit-unchanged; the head equals torch's clip_grad_norm_(0.1) +
    AdamW over the head alone fed the engine's gradients (fp32, rtol 1e-5 as in test_clip_and_adamw_vs_torch)."""
    rotated = True
    grid, gt = _planted(DIMS, 12, 11, rotated)
    grid, gt = grid.cuda()[None], [gt.cuda()]
    eng = _engine((2, 1, 1, 1), rotated, precision, True, lr=3e-4, weight_decay=0.01, clip_grad_norm=0.1)
    lo = eng.head_lo
    bb0 = [t[:lo].clone() for t in (eng.flat_p, eng.flat_m, eng.flat_v)]
    q = torch.nn.Parameter(eng.flat_p[lo:].clone())
    opt = torch.optim.AdamW([q], lr=3e-4, weight_decay=0.01)
    clipped = 0
    for step in range(4):
        eng.forward_backward(grid, gt)
        torch.cuda.synchronize()
        q.grad = eng.flat_g[lo:] / eng.loss_scale
        tn = torch.nn.utils.clip_grad_norm_([q], 0.1)
        clipped += int(tn.item() > 0.1)
        opt.step()
        eng.optimizer_step()
        torch.cuda.synchronize()
        assert abs(eng._norm.item() - tn.item()) <= 1e-5 * tn.item()
        assert torch.allclose(eng.flat_p[lo:], q.data, rtol=1e-5, atol=1e-7), (step, (eng.flat_p[lo:] - q.data).abs().max().item())
        for a, b in zip((eng.flat_p, eng.flat_m, eng.flat_v), bb0):
            assert torch.equal(a[:lo], b)
    # the head's 16-bit operands follow the updated master weights (the backbone's are the ones packed at construction)
    from nerf_rpn_b200 import packing
    for layer in eng.hconv:
        want, _ = packing.pack_conv_weight(layer.weight.data.cpu(), dtype=eng.act_dtype)
        assert torch.equal(layer.fwd.cpu(), want)
    print(f"[{precision}] {clipped} of 4 steps clipped")


# ------------------------------------------------------------------------------------------------ 4. memory
def _backbone_grad_bytes(layers, dims, elem=2):
    """Bytes of the full plan's backbone and FPN gradient buffers: dp0, da0, dy0, every block's dout, dq[0..3] and the smooth convs' df."""
    from nerf_rpn_b200.engine import _down

    def vol(d):
        return d[0] * d[1] * d[2]
    d1 = _down(dims); d2 = _down(d1)
    total = vol(d2) * 64 + 2 * vol(d1) * 64
    xd, stage_dims = d2, []
    for si, nb in enumerate(layers):
        od = xd if si == 0 else _down(xd)
        total += nb * vol(od) * 64 * 2 ** si * 4
        stage_dims.append(od)
        xd = od
    total += sum(vol(d) * 256 for d in stage_dims) + sum(vol(d) * 256 for d in stage_dims[:3])
    return total * elem


def test_frozen_plan_pool_does_not_grow_with_depth():
    def pool(layers, frozen):
        eng = _engine(layers, True, "bf16", frozen)
        eng.plan(1, DIMS)
        return eng.cache_stats()["pool_bytes"]
    deep_z, shallow_z = pool((3, 4, 6, 3), True), pool((2, 1, 1, 1), True)
    deep_f, shallow_f = pool((3, 4, 6, 3), False), pool((2, 1, 1, 1), False)
    print(f"pool bytes at {DIMS}: frozen {deep_z / 2**20:.1f} / {shallow_z / 2**20:.1f} MiB, full {deep_f / 2**20:.1f} / {shallow_f / 2**20:.1f} MiB "
          f"((3,4,6,3) / (2,1,1,1))")
    assert deep_z == shallow_z and deep_f != shallow_f
    for layers, z, f in (((3, 4, 6, 3), deep_z, deep_f), ((2, 1, 1, 1), shallow_z, shallow_f)):
        assert z <= f - _backbone_grad_bytes(layers, DIMS), (layers, z, f, _backbone_grad_bytes(layers, DIMS))


# ------------------------------------------------------------------------------------------------ 5. the drop-in loop
def test_dropin_loop_frozen_backbone_then_unfrozen():
    """run_rpn.py:384-395 with --freeze_backbone (weights, reg_loss_weight scaling, clip_grad_norm_, torch AdamW, zero_grad) equals the same loop
    on the full step with the backbone's gradients discarded, bit for bit, and leaves the backbone's weights unchanged; after unfreezing, one
    more step gives the backbone gradients, equal to the full step's."""
    rotated = True
    batches = [_planted(DIMS, 12, 30 + k, rotated) for k in range(4)]
    batches = [([g.cuda()], [t.cuda()]) for g, t in batches]
    a, b = _model((2, 1, 1, 1), rotated), _model((2, 1, 1, 1), rotated)
    for p in a.backbone.parameters():
        p.requires_grad = False
    bb0 = [p.detach().clone() for p in a.backbone.parameters()]
    opts = [torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0.01) for m in (a, b)]

    def step(m, opt, batch, seed, discard_backbone):
        torch.manual_seed(seed)
        _, losses, _ = m(*batch)
        losses["loss_rpn_box_reg"] *= 5.0
        losses["loss_rpn_box_reg_2d"] *= 0.0
        loss = losses["loss_objectness"] + losses["loss_rpn_box_reg"] + losses["loss_rpn_box_reg_2d"]
        loss.backward()
        if discard_backbone:
            for p in m.backbone.parameters():
                p.grad = None
        grads = [None if p.grad is None else p.grad.clone() for p in m.parameters()]
        torch.nn.utils.clip_grad_norm_(m.parameters(), 0.1)
        opt.step()
        opt.zero_grad()
        return loss.detach(), grads

    for k, batch in enumerate(batches):
        la, ga = step(a, opts[0], batch, 100 + k, False)
        lb, gb = step(b, opts[1], batch, 100 + k, True)
        assert a.train_engine().plan_for(batch[0]).frozen and not b.train_engine().plan_for(batch[0]).frozen
        assert torch.equal(la, lb), (k, la.item(), lb.item())
        for x, y in zip(ga, gb):
            assert (x is None and y is None) or torch.equal(x, y)
        for x, y in zip(a.rpn.head.parameters(), b.rpn.head.parameters()):
            assert torch.equal(x, y)
    assert all(torch.equal(p, q) for p, q in zip(a.backbone.parameters(), bb0))
    assert any(not torch.equal(p, q) for p, q in zip(a.rpn.head.parameters(), _model((2, 1, 1, 1), rotated).rpn.head.parameters()))
    # unfreeze: the next forward runs the full step and the backbone's gradients come back
    for p in a.backbone.parameters():
        p.requires_grad = True
    la, ga = step(a, opts[0], batches[0], 200, False)
    lb, gb = step(b, opts[1], batches[0], 200, False)
    assert not a.train_engine().plan_for(batches[0][0]).frozen
    assert torch.equal(la, lb)
    n_bb = len(list(a.backbone.parameters()))
    assert all(g is not None for g in ga[:n_bb])
    for x, y in zip(ga, gb):
        assert torch.equal(x, y)

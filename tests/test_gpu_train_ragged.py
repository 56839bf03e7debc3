"""GPU: training on batches of differently sized scenes (the reference pads a batch to its element-wise maximum, nerf_rpn.py:129-146, and
labels the anchors in the padding -1, anchor.py:124-152 / rpn.py:231-238, 260-263, 283-285) and the engine's bounded plan pool.
Reference pieces come from the staged oracle/_ref only."""
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_train import _grad_metrics, _planted

pytestmark = pytest.mark.gpu


def _scene(dims, seed, channels_last):
    """A (4,X,Y,Z) fp32 CUDA scene with RGB in [0,1) and raw densities N(2, 3); contiguous or the dataset's channels-last view."""
    g = torch.Generator().manual_seed(seed)
    raw = torch.rand(*dims, 4, generator=g)
    raw[..., 3] = torch.randn(*dims, generator=g) * 3.0 + 2.0
    raw = raw.cuda()
    return raw.permute(3, 0, 1, 2) if channels_last else raw.permute(3, 0, 1, 2).contiguous()


def _alpha(s):
    """datasets.py:165-167 on the device with torch: clip(1 - exp(-exp(sigma) / 100), 0, 1) of the density channel."""
    out = s.clone()
    out[3] = torch.clamp(1.0 - torch.exp(-torch.exp(s[3]) / 100.0), 0.0, 1.0)
    return out


def _pad_stack(scenes, value_density=0.0):
    X, Y, Z = (max(int(s.shape[1 + a]) for s in scenes) for a in range(3))
    out = []
    for s in scenes:
        p = (0, Z - s.shape[3], 0, Y - s.shape[2], 0, X - s.shape[1])
        rgb = F.pad(s[:3].contiguous(), p, value=0.0)
        d = F.pad(s[3:].contiguous(), p, value=value_density)
        out.append(torch.cat([rgb, d], 0))
    return torch.stack(out, 0)


# ------------------------------------------------------------------------------------------------ engine helpers
def _model(layers, rotated, ref_state=None, alpha=False):
    from oracle import ref_gpu
    from nerf_rpn_b200.model.anchor import AnchorGenerator3D, RPNHead
    from nerf_rpn_b200.model.feature_extractor import Bottleneck, ResNet_FPN_256
    from nerf_rpn_b200.model.nerf_rpn import NeRFRegionProposalNetwork
    torch.manual_seed(0)
    backbone = ResNet_FPN_256(Bottleneck, list(layers), input_dim=4, is_max_pool=True)
    head = RPNHead(256, 13, 4, rotate=rotated)
    if ref_state is not None:
        backbone.load_state_dict(ref_state["bsd"]); head.load_state_dict(ref_state["hsd"])
    return NeRFRegionProposalNetwork(backbone, AnchorGenerator3D(ref_gpu.ANCHOR_SIZES, ref_gpu.ASPECT), head, rpn_fg_iou_thresh=0.35,
                                     rpn_bg_iou_thresh=0.2, rotated_bbox=rotated, density_to_alpha_on_device=alpha).cuda().train()


def _need_ref():
    from oracle import ref_gpu
    if not ref_gpu.available():
        pytest.skip("oracle/_ref not staged")
    return ref_gpu


def _batch(dims_list, n_gt, rotated, seed=11):
    grids, gts = [], []
    for i, d in enumerate(dims_list):
        g, t = _planted(d, n_gt, seed + i, rotated)
        grids.append(g.cuda()); gts.append(t.cuda())
    return grids, gts


# ------------------------------------------------------------------------------------------------ 2. masks and labels
def test_padding_mask_and_labels_vs_reference():
    ref_gpu = _need_ref()
    from nerf_rpn_b200 import ops
    from nerf_rpn_b200.train import RPNTrainEngine
    dims_list = [(48, 64, 40), (36, 56, 52)]
    grids, gts = _batch(dims_list, 10, False)
    gts[1] = gts[1][:0]                                            # the second scene has no ground truth
    m = ref_gpu.build_reference_model(rotated=False, seed=0, layers=(2, 1, 1, 1), rpn_fg_iou_thresh=0.35, rpn_bg_iou_thresh=0.2).cuda()
    eng = RPNTrainEngine(_model((2, 1, 1, 1), False), precision="bf16")
    plan = eng.plan_for(grids)
    meshes = _pad_stack(grids)
    feats = [torch.empty((2, 1, *d), device="cuda") for d in plan.feat_dims]
    want_mask = m.rpn.get_padding_masks(meshes, feats, [torch.Size(d) for d in dims_list])
    plan._set_input(grids)
    got_mask = plan.padding_masks()
    assert got_mask is not None and torch.equal(got_mask.bool(), want_mask)
    assert (~want_mask[0]).any() and (~want_mask[1]).any()
    anchors_ref = [a.cuda() for a in m.rpn.anchor_generator(meshes, feats)[0]]
    anchors = plan._anchors()
    assert torch.equal(anchors, anchors_ref[0])
    labels_ref, matched_ref = m.rpn.assign_targets_to_anchors(anchors_ref, gts, want_mask)
    lab0, idx0 = ops.assign_targets(anchors, gts[0], got_mask[0], 0.35, 0.2, True)
    assert torch.equal(lab0, labels_ref[0])
    assert torch.equal(gts[0][idx0.clamp(min=0)], matched_ref[0])
    assert (lab0 == 1).sum() > 0 and (lab0[~got_mask[0].bool()] == -1).all()
    # the background scene through the engine's own forward: no positives, and every sampled negative lies inside the scene
    torch.manual_seed(3)
    plan.forward_loss(grids, gts)
    pos1, neg1, _ = plan.last_samples[1]
    assert pos1.numel() == 0 and neg1.numel() == 256
    assert got_mask[1][neg1].all()
    assert ((labels_ref[1] == 0) == got_mask[1].bool()).all() and (labels_ref[1][~got_mask[1].bool()] == -1).all()


# ------------------------------------------------------------------------------------------------ 3. training step
def _reference_batch_step(ref_gpu, rotated, layers, grids, gts, autocast_dtype=None):
    m = ref_gpu.build_reference_model(rotated=rotated, seed=0, layers=layers, rpn_fg_iou_thresh=0.35, rpn_bg_iou_thresh=0.2).cuda().train()
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
        _, losses, _ = m(list(grids), list(gts))                  # a copy: the reference pads the list in place
        loss = losses["loss_objectness"] + 5.0 * losses["loss_rpn_box_reg"]
    loss.backward()
    params = list(m.backbone.parameters()) + list(m.rpn.head.parameters())
    out["names"] = [n for n, _ in m.backbone.named_parameters()] + ["head." + n for n, _ in m.rpn.head.named_parameters()]
    out["grads"] = [p.grad.detach().float().clone() for p in params]
    out["losses"] = (losses["loss_objectness"].item(), losses["loss_rpn_box_reg"].item())
    out["samples"] = list(zip(rec["pos"], rec["neg"]))
    del m
    torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize("layers,rotated,precision", [((2, 1, 1, 1), False, "bf16"), ((2, 1, 1, 1), True, "fp16"), ((3, 4, 6, 3), True, "bf16")])
def test_ragged_training_step_vs_reference_autograd(layers, rotated, precision):
    """Two differently sized scenes, trained as the reference trains their padded batch; the criteria and the mixed-precision baseline of
    test_gpu_train.test_training_step_vs_reference_autograd (the engine is held to the reference's own autocast run against fp32)."""
    ref_gpu = _need_ref()
    from nerf_rpn_b200.train import RPNTrainEngine
    grids, gts = _batch([(64, 96, 80), (56, 80, 72)], 12, rotated)
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
    try:
        r32 = _reference_batch_step(ref_gpu, rotated, layers, grids, gts)
        rac = _reference_batch_step(ref_gpu, rotated, layers, grids, gts, torch.bfloat16 if precision == "bf16" else torch.float16)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    model = _model(layers, rotated, r32)
    eng = RPNTrainEngine(model, precision=precision, lr=1e-4, weight_decay=0.01, clip_grad_norm=0.1, reg_loss_weight=5.0)
    torch.manual_seed(123)
    out = eng.forward_backward(grids, gts)
    torch.cuda.synchronize()
    plan = eng.plan_for(grids)
    assert plan.dims == (64, 96, 80) and plan.valid is not None
    same = all(set(p.tolist()) == set(rp.tolist()) and set(q.tolist()) == set(rq.tolist())
               for (p, q, _), (rp, rq) in zip(plan.last_samples, r32["samples"]))
    got_l = out.tolist()
    inv = 1.0 / eng.loss_scale
    params = list(model.backbone.parameters()) + list(model.rpn.head.parameters())
    grads = [eng.grad_of(p).view(p.shape).clone() * inv for p in params]
    cos_o, rel_o, per_o = _grad_metrics(grads, r32)
    cos_a, rel_a, per_a = _grad_metrics(rac["grads"], r32)
    tag = f"[ragged {layers} {'OBB' if rotated else 'AABB'} {precision}]"
    print(f"{tag} sampler reproduces the reference's draws for both scenes: {same}")
    print(f"{tag} losses: ours {got_l}  reference fp32 {r32['losses']}  reference autocast {rac['losses']}")
    print(f"{tag} gradient vs reference fp32: ours cosine {cos_o:.4f} rel {rel_o:.3f} | reference autocast cosine {cos_a:.4f} rel {rel_a:.3f}")
    checks = [(same, "the sampler did not reproduce the reference's draws")]
    for k in range(2):
        e_o, e_a = abs(got_l[k] - r32["losses"][k]), abs(rac["losses"][k] - r32["losses"][k])
        slack = (1e-2 if precision == "bf16" else 3e-3) * abs(r32["losses"][k])
        checks.append((e_o <= 3.0 * e_a + slack, f"loss {k}: ours off by {e_o}, autocast by {e_a}"))
    checks.append((cos_o >= cos_a - 0.08, f"gradient cosine {cos_o} vs autocast {cos_a}"))
    checks.append((rel_o <= 1.15 * rel_a + 0.02, f"gradient rel err {rel_o} vs autocast {rel_a}"))
    bad = [(n, v, per_a[n]) for n, v in per_o.items() if v > 1.25 * per_a[n] + 0.03]
    checks.append((not bad, f"tensors worse than the autocast reference: {bad[:5]}"))
    if tuple(layers) == (2, 1, 1, 1):
        checks.append((cos_o >= (0.98 if precision == "fp16" else 0.80), f"shallow network: gradient cosine {cos_o}"))
    failed = [msg for ok, msg in checks if not ok]
    assert not failed, failed


# ------------------------------------------------------------------------------------------------ 4. drop-in
def test_dropin_ragged_batch_gradients_equal_engine():
    model = _model((2, 1, 1, 1), True)
    a, b = _scene((40, 56, 48), 1, True), _scene((48, 40, 36), 2, False)
    a[3].clamp_(0, 1); b[3].clamp_(0, 1)
    (_, ga), (_, gb) = _planted((40, 56, 48), 6, 3, True), _planted((48, 40, 36), 6, 4, True)
    ga, gb = ga.cuda(), gb.cuda()
    meshes = [a, b]
    torch.manual_seed(5)
    _, losses, _ = model(meshes, [ga, gb])
    assert meshes[0] is a and meshes[1] is b and a.shape == (4, 40, 56, 48)          # the caller's list is not padded in place
    assert all(v.grad_fn is not None for v in losses.values())
    (losses["loss_objectness"] + 5.0 * losses["loss_rpn_box_reg"]).backward()
    params = list(model.backbone.parameters()) + list(model.rpn.head.parameters())
    got = [p.grad.clone() for p in params]
    eng = model.train_engine()
    plan = eng.plan_for(meshes)
    plan.forced_samples = [(p, q) for p, q, _ in plan.last_samples]
    try:
        eng.forward_backward(meshes, [ga, gb])
    finally:
        del plan.forced_samples
    torch.cuda.synchronize()
    inv = 1.0 / eng.loss_scale
    for p, g in zip(params, got):
        e = eng.grad_of(p).view(p.shape)
        assert torch.equal(g, e * inv if inv != 1.0 else e)


# ------------------------------------------------------------------------------------------------ 5. bounded memory
def test_plan_pool_memory_bounded_over_many_shapes():
    from nerf_rpn_b200 import train as T
    eng = T.RPNTrainEngine(_model((2, 1, 1, 1), True), precision="bf16")
    largest = [(48, 64, 48), (40, 56, 44)]
    others = [[(48 - 4 * i, 60 - 2 * i, 40), (32, 48 - 2 * i, 44 - 3 * (i % 3))] for i in range(11)]
    shapes = [largest] + others
    assert len({tuple(max(s[a] for s in b) for a in range(3)) for b in shapes}) == 12
    batches = []
    for k, b in enumerate(shapes):
        grids, gts = _batch(b, 6, True, seed=100 + 3 * k)
        batches.append((grids, gts))
    params = list(eng.model.backbone.parameters()) + list(eng.model.rpn.head.parameters())

    def step(k):
        torch.manual_seed(77)
        losses = eng.forward_backward(*batches[k]).clone()
        torch.cuda.synchronize()
        return losses, torch.cat([eng.grad_of(p) for p in params]).clone()

    first = [step(0) for _ in range(3)]                        # fresh plan, second eager run, captured graph
    res_first = torch.cuda.max_memory_reserved()
    growths = eng.cache_stats()                                 # the first backward pass sizes its scratch buffers block by block
    for k in range(1, len(shapes)):
        for _ in range(3):
            step(k)
        st = eng.cache_stats()
        assert st["plans"] <= T.PLAN_CACHE and st["graphs"] <= 2 * T.PLAN_CACHE, st
    again = [step(0) for _ in range(3)]                        # rebuilt after eviction: eager twice, then a new graph
    res_end = torch.cuda.max_memory_reserved()
    st = eng.cache_stats()
    print(f"max_memory_reserved after the first shape {res_first / 2**20:.1f} MiB, after 12 shapes {res_end / 2**20:.1f} MiB; {st}")
    assert st["plans"] <= T.PLAN_CACHE and st["graphs"] >= 1
    assert st["pool_growths"] == growths["pool_growths"] and st["scratch_growths"] == growths["scratch_growths"], "a smaller batch grew the pool"
    for (l0, g0), (l1, g1) in zip(first + again, [first[0]] * 6):
        assert torch.equal(l0, l1) and torch.equal(g0, g1)
    assert res_end <= 1.10 * res_first + (64 << 20), (res_first, res_end)


# ------------------------------------------------------------------------------------------------ 6. density_to_alpha in training
@pytest.mark.parametrize("ragged", [False, True])
def test_training_density_to_alpha_on_device(ragged):
    from nerf_rpn_b200.train import RPNTrainEngine
    model = _model((2, 1, 1, 1), False)
    eng = RPNTrainEngine(model, precision="bf16")
    dims = [(40, 48, 36), (32, 48, 40)] if ragged else [(40, 48, 36), (40, 48, 36)]
    raw = [_scene(d, 20 + i, i == 0) for i, d in enumerate(dims)]
    for s in raw:      # densities far from 0 map to exactly 0 or 1 in any fp32 exp, so the host map below has the kernel's bits
        s[3] = torch.where(s[3] > 2.0, 12.0 + s[3], -30.0 + s[3])
    mapped = [_alpha(s) for s in raw]
    assert all(((m[3] == 0) | (m[3] == 1)).all() for m in mapped)
    gts = [_planted(d, 6, 30 + i, False)[1].cuda() for i, d in enumerate(dims)]

    def losses(grids, flag):
        model.density_to_alpha_on_device = flag
        torch.manual_seed(9)
        plan = eng.plan_for(grids)
        plan.forward_loss(grids, gts)
        torch.cuda.synchronize()
        return eng.losses.clone()

    if ragged:
        on, off = losses(raw, True), losses(mapped, False)
    else:
        on = losses(torch.stack([s.contiguous() for s in raw]), True)
        off = losses(torch.stack([s.contiguous() for s in mapped]), False)
    raw_only = losses(raw if ragged else torch.stack([s.contiguous() for s in raw]), False)
    assert torch.equal(on, off), (on, off)
    assert not torch.equal(on, raw_only)                       # the flag is honoured: raw densities give other losses


# ------------------------------------------------------------------------------------------------ 7. pool growth frees what it replaces
def test_pool_growth_frees_replaced_slots_and_evicted_plans():
    """small batch -> larger batch (every slot grows, the small plan is dropped) -> small again.  With the cyclic collector OFF, the replaced
    slots and the dropped plan must be gone at once (a plan's launch lists are closures over it), and the allocated memory must be the pool,
    the shared scratch and the cached anchors -- no second copy of the old slots."""
    import gc
    import weakref
    from nerf_rpn_b200 import train as T
    eng = T.RPNTrainEngine(_model((2, 1, 1, 1), True), precision="bf16")
    small, large = _batch([(40, 48, 40), (32, 48, 36)], 6, True, seed=50), _batch([(64, 80, 72), (56, 72, 64)], 6, True, seed=60)
    gc.collect()                                                # earlier engines (a model and its engine refer to each other)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    gc.disable()
    try:
        for _ in range(3):                                       # eager, eager, captured graphs
            eng.forward_backward(*small)
        torch.cuda.synchronize()
        st0 = eng.cache_stats()
        assert st0["graphs"] == 2
        old_slots = [weakref.ref(t) for t in eng._pool]
        old_plan = weakref.ref(eng.plan_for(small[0]))
        for _ in range(3):
            eng.forward_backward(*large)
        torch.cuda.synchronize()
        st1 = eng.cache_stats()
        assert st1["pool_growths"] == st0["pool_growths"] + 1 and st1["plans"] == 1 and st1["pool_bytes"] > 2 * st0["pool_bytes"]
        assert old_plan() is None, "the dropped plan is still alive"
        replaced = [r for r in old_slots if not any(r() is t for t in eng._pool)]
        assert replaced and all(r() is None for r in replaced), "a replaced pool slot is still referenced"
        extra = torch.cuda.memory_allocated() - base - st1["pool_bytes"] - st1["scratch_bytes"] - st1["anchor_bytes"]
        print(f"pool {st0['pool_bytes'] / 2**20:.1f} -> {st1['pool_bytes'] / 2**20:.1f} MiB, scratch {st1['scratch_bytes'] / 2**20:.1f} MiB, "
              f"anchors {st1['anchor_bytes'] / 2**20:.1f} MiB, other allocations {extra / 2**20:.1f} MiB")
        assert abs(extra) < 16 << 20 and extra < st0["pool_bytes"] / 2, "allocated memory is not the pool, scratch and anchors"
        # the small batch again fits in the grown pool: nothing grows, both plans stay cached
        for _ in range(3):
            eng.forward_backward(*small)
        torch.cuda.synchronize()
        st2 = eng.cache_stats()
        assert st2["pool_growths"] == st1["pool_growths"] and st2["pool_bytes"] == st1["pool_bytes"] and st2["plans"] == 2
        # least-recently-used eviction frees the evicted plan at once as well
        lru = weakref.ref(eng.plan_for(large[0]))
        for k in range(T.PLAN_CACHE):
            eng.forward_backward(*_batch([(36 - 2 * k, 44, 36), (20, 40, 36)], 4, True, seed=70 + k))      # four new padded shapes
        assert lru() is None and eng.cache_stats()["plans"] == T.PLAN_CACHE
    finally:
        gc.enable()


# ------------------------------------------------------------------------------------------------ 8. one forward at a time
def test_dropin_second_forward_before_backward_raises():
    """Every batch shape trains in the engine's one set of buffers: a backward after a later forward would read overwritten activations, so it
    raises instead of returning wrong gradients."""
    model = _model((2, 1, 1, 1), True)
    a, b = _batch([(40, 48, 40), (32, 48, 36)], 6, True, seed=80), _batch([(48, 40, 36), (40, 40, 40)], 6, True, seed=90)
    _, l1, _ = model(*a)
    _, l2, _ = model(*b)
    with pytest.raises(RuntimeError, match="another training forward"):
        (l1["loss_objectness"] + l2["loss_objectness"]).backward()
    _, l3, _ = model(*a)                                       # forward / backward pairs keep working
    (l3["loss_objectness"] + 5.0 * l3["loss_rpn_box_reg"]).backward()
    assert all(p.grad is not None for p in model.backbone.parameters())

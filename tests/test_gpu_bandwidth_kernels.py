"""The training step's bandwidth kernels (csrc/train.cu: BatchNorm statistics / apply / backward, max-pool 3/2/1 with argmax and its
backward, nearest up-sampling backward, stride-2 gather / scatter, gradient accumulation, RPN loss, weight packing, gradient norm and
clip + AdamW) and the VGG pooling and stride-1 stem packing of csrc/pointwise.cu, against the float64 references of tests/emulate.py
in both 16-bit activation formats.

One table of named rows.  Every row draws its operands from a generator seeded by the row's name and checks:
  - nothing unwritten, nothing over-written: outputs sit inside NaN guard bands (GUARD elements before and after) and are NaN-filled,
    or hold their pre-existing value where the kernel adds into them (the coarse gradient of the up-sampling, the running statistics,
    the optimiser state).  Afterwards every element the kernel must write is finite and within bound and every other element keeps
    its bits: the guard bands, and the whole predictor gradient around the sampled anchors of the RPN loss;
  - a per-element bound, with u = half an ulp of the 16-bit output format (2^-8 bf16, 2^-11 fp16) and e = 2^-24:

  BN statistics   k = ceil(ceil(rows / B) / lanes) + lanes, the longest fp32 chain of chan_reduce_kernel (B = min(rows, 296) blocks,
                  lanes = max(256 / (C / 8), 1) rows per pass; each thread sums its rows, then the lanes are added one by one; only
                  the 296 block partials are summed in fp64).  The fp32 sums of y and y^2 are off by at most k e of sum |y| and of
                  sum y^2, so  |mean - ref| <= (k + 2) e E|y|  and the variance E[y^2] - mean^2 by at most 3 (k + 2) e E[y^2]:
                  |rstd - ref| <= rstd (1.5 (k + 2) e E[y^2] / (var + eps) + 2e).  The statistics term grows with mean^2 / var
                  (E[y^2] / var = 1 + mean^2 / var): it is the cancellation of the one-pass variance.  The running statistics
                  carry momentum times these errors (the variance times rows / (rows - 1)) and one fp32 rounding.
  BN apply        |got - ref| <= u |ref| + 8 e (|gamma x_hat| + |beta| + |res|) + e, on the fp32 statistics the kernel read:
                  five fp32 operations, then one 16-bit rounding (ReLU is 1-Lipschitz).
  BN backward     dgamma, dbeta: the same chain, (k + 4) e sum |g x_hat| and (k + 1) e sum |g|, plus one fp32 rounding.
                  dy: u |ref| + 10 e |gamma rstd| (|g| + |dbeta| / M + |x_hat dgamma| / M) + e, on the sums the kernel read.
                  dres = g exactly (u |ref| + e).
  max-pool        forward and argmax exact; backward: a sum of <= 8 16-bit values in fp32, u |ref| + 8 e sum |dy| + e.
  up-sampling     the existing coarse value plus T fine values in fp32 (T the largest pre-image): u |ref| + (T + 1) e mag + e.
  RPN loss        targets: 16 e tmag, tmag = (|coordinates| and sizes read) / smallest size + |t| + 1 (the encoders' fp32 rounding of
                  box coordinates, divided by a box size).  dlogit: u |ref| + 8 e K + e, K = w_obj grad_scale / norm (expf, the
                  reciprocal and three products).  ddelta: u |ref| + 9 K_r (dt + 2 e (|p| + |t|)) + e, 9 = 1/beta the smooth-L1
                  gradient's Lipschitz constant, dt the target bound.  Losses: the same per-term errors summed over the terms / norm,
                  plus e of the accumulated value per call.
  grad norm       fp64 sums of exact fp32 squares: 2^-22 of the norm.
  AdamW           on the fp32 hyper-parameters and the fp32 norm the kernel read: e-multiples of each fp32 operation, and the host's
                  fp32 bias corrections 1 - b^t, whose relative error is e (b^t / (1 - b^t) + 1) (1e3 e for b2 = 0.999 at t = 1).
  layouts         stride-2 gather / scatter, max-pool outputs, weight packing, stride-1 stem packing: bit for bit after one 16-bit
                  rounding.
tests/test_bandwidth_reference_cpu.py checks the references against torch in float64 and that each bound, on the reference's own
scale, rejects a reference with one deliberate mistake by at least 4x on the row aimed at it.
test_table_covers_every_path records the launches of real training steps and inference forwards and asserts that a row covers each
(entry point, channel count, flags, dtype) combination.  Run with -s to see the worst err / bound of every row."""
import ctypes
import dataclasses
import math
import zlib
from typing import Optional, Tuple

import numpy as np
import pytest
import torch

from tests.emulate import (emulate_pack_stem_s1, encode_targets64, reference_adamw64, reference_bn_apply64, reference_bn_backward64,
                           reference_bn_stats64, reference_grad_norm64, reference_maxpool2_ceil, reference_maxpool3_argmax,
                           reference_maxpool3_backward64, reference_rpn_loss64, reference_upsample_backward64, rpn_anchors_f32)

pytestmark = pytest.mark.gpu

DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}
HALF_ULP = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
E = 2.0 ** -24
GUARD = 64
EPS = 1e-5
RED_BLOCKS = 296
CHUNK = 1 << 18                                  # rows per float64 reference slice of the 1.3 M-row BatchNorms
HEAD_LO = 52_514_176                             # ResNet50-FPN backbone parameters: the head's offset in the flat buffers
HEAD_N = {True: 7_108_981, False: 7_102_299}     # rotated / axis-aligned RPN head parameters


@dataclasses.dataclass(frozen=True)
class BN:
    c: int
    rows: int
    dtype: str = "bf16"
    kind: str = "residual"                       # "residual": ReLU + res + dres; "relu": ReLU only; "plain": neither (downsample BN)
    mean: float = 0.3
    std: float = 1.5
    running: bool = True                         # random running statistics (False: 0 and 1, a fresh module)


@dataclasses.dataclass(frozen=True)
class Pool:
    dims: Tuple[int, int, int]
    c: int = 64
    n: int = 1
    dtype: str = "bf16"
    post_relu: bool = True                       # relu(randn - 2): most windows of zeros, ties decided by the first-maximum rule


@dataclasses.dataclass(frozen=True)
class Pool2:
    dims: Tuple[int, int, int]
    c: int
    n: int = 1
    dtype: str = "bf16"


@dataclasses.dataclass(frozen=True)
class Up:
    fine: Tuple[int, int, int]
    coarse: Tuple[int, int, int]
    c: int = 256
    n: int = 1
    dtype: str = "bf16"


@dataclasses.dataclass(frozen=True)
class Stride2:
    dims: Tuple[int, int, int]
    c: int
    n: int = 1
    dtype: str = "bf16"


@dataclasses.dataclass(frozen=True)
class Pack:
    cout: int
    cin: int
    k: int
    dtype: str = "bf16"
    bwd: bool = True


@dataclasses.dataclass(frozen=True)
class StemS1:
    dims: Tuple[int, int, int]
    n: int = 1
    dtype: str = "bf16"


@dataclasses.dataclass(frozen=True)
class Loss:
    rotated: bool
    dtype: str = "fp16"
    n_pos: Tuple[int, ...] = (100,)              # one call per entry (a batch accumulating into one losses pair)
    n_neg: Tuple[int, ...] = (150,)
    w_reg: float = 5.0
    theta: Optional[Tuple[float, ...]] = None    # the angles the positives' boxes cycle through (random in (-pi/2, pi/2) if None)


@dataclasses.dataclass(frozen=True)
class Opt:
    n: int
    offset: int = 0                              # floats before the range (a frozen engine's head_lo; 1 reaches the unaligned path)
    inv_scale: float = 1.0
    max_norm: float = 0.1
    steps: Tuple[int, ...] = (1,)
    grad_std: Tuple[float, ...] = (1e-5,)        # per step
    warm: bool = False                           # random m, v (a later step) instead of zeros


D4 = {"stem": (80, 128, 128), "s1": (40, 64, 64), "s2": (20, 32, 32), "s3": (10, 16, 16), "s4": (5, 8, 8)}     # config 4, 160x256x256
DS = {"stem": (32, 48, 40), "s1": (16, 24, 20), "s2": (8, 12, 10), "s3": (4, 6, 5), "s4": (2, 3, 3)}         # (2,1,1,1) at 64x96x80
DR = {"stem": (24, 32, 66), "s1": (12, 16, 33), "s2": (6, 8, 17), "s3": (3, 4, 9), "s4": (2, 2, 5)}          # ragged n = 2, P2 depth 33
VGG = ((32, 32, 32), (16, 16, 16), (8, 8, 8), (4, 4, 4))


def _vol(d):
    return d[0] * d[1] * d[2]


def _bn_rows():
    """Every BatchNorm the engine launches, at the row counts of config 4, the ragged batch and the (2,1,1,1) test model: the stem
    (ReLU), each stage's narrow bn1 / bn2 (ReLU), its wide bn3 (residual + ReLU, skip-branch gradient) and downsample BN (neither)."""
    rows = {}
    for dt in ("bf16", "fp16"):
        for name, dims, n in (("c4", D4, 1), ("ragged", DR, 2), ("small", DS, 1)):
            rows[f"bn_{name}_stem_c64_relu_{dt}"] = BN(64, n * _vol(dims["stem"]), dt, "relu")
            for stage, narrow in (("s1", 64), ("s2", 128), ("s3", 256), ("s4", 512)):
                r = n * _vol(dims[stage])
                rows[f"bn_{name}_{stage}_c{narrow}_relu_{dt}"] = BN(narrow, r, dt, "relu")
                rows[f"bn_{name}_{stage}_c{4 * narrow}_residual_{dt}"] = BN(4 * narrow, r, dt, "residual")
                rows[f"bn_{name}_{stage}_c{4 * narrow}_plain_{dt}"] = BN(4 * narrow, r, dt, "plain")
    rows.update({
        "bn_mean30_c64_fp16": BN(64, _vol(DS["stem"]), "fp16", "relu", mean=30.0, std=1.0),
        "bn_mean30_c256_bf16": BN(256, 7680, "bf16", "plain", mean=-30.0, std=1.0),
        "bn_mean30_c2048_fp16": BN(2048, 18, "fp16", "residual", mean=30.0, std=1.0),
        "bn_c64_fresh_running_bf16": BN(64, 40 * 64 * 16, "bf16", running=False),
        "bn_c256_5000_fp16": BN(256, 5000, "fp16"),
        "bn_c2048_333_bf16": BN(2048, 333, "bf16"),
        "bn_c96_1000_fp16": BN(96, 1000, "fp16"),                                   # 12 channel groups: constants reloaded per chunk
        "bn_c96_1000_plain_bf16": BN(96, 1000, "bf16", "plain"),
        "bn_c64_rows3_fp16": BN(64, 3, "fp16", "plain"),                             # 3 blocks of one row
    })
    return rows


ROWS = dict(_bn_rows())
for _dt in ("bf16", "fp16"):
    ROWS.update({
        f"pool_c4_stem_{_dt}": Pool(D4["stem"], dtype=_dt),
        f"pool_small_stem_{_dt}": Pool(DS["stem"], dtype=_dt),
        f"pool_ragged_stem_n2_{_dt}": Pool(DR["stem"], n=2, dtype=_dt),
        f"pool_odd_c16_n2_randn_{_dt}": Pool((16, 8, 7), 16, 2, _dt, post_relu=False),
        f"pool_9x12x10_n2_randn_{_dt}": Pool((9, 12, 10), 64, 2, _dt, post_relu=False),
        f"up_c4_p4_{_dt}": Up(D4["s3"], D4["s4"], dtype=_dt),
        f"up_c4_p3_{_dt}": Up(D4["s2"], D4["s3"], dtype=_dt),
        f"up_c4_p2_{_dt}": Up(D4["s1"], D4["s2"], dtype=_dt),
        f"up_ragged_p2_n2_{_dt}": Up(DR["s1"], DR["s2"], n=2, dtype=_dt),
        f"up_ragged_p3_n2_{_dt}": Up(DR["s2"], DR["s3"], n=2, dtype=_dt),
        f"up_ragged_p4_n2_{_dt}": Up(DR["s3"], DR["s4"], n=2, dtype=_dt),
        f"up_small_p2_{_dt}": Up(DS["s1"], DS["s2"], dtype=_dt),
        f"up_46_from_14_{_dt}": Up((46, 9, 7), (14, 5, 4), c=8, dtype=_dt),       # float32 and float64 nearest indices differ
        f"up_13x9x7_c64_{_dt}": Up((13, 9, 7), (7, 5, 4), c=64, dtype=_dt),
        f"up_25x25x17_c64_{_dt}": Up((25, 25, 17), (13, 13, 9), c=64, dtype=_dt),
        f"stride2_9x12x7_c128_n2_{_dt}": Stride2((9, 12, 7), 128, 2, _dt),
        f"stride2_ragged_s1_c256_n2_{_dt}": Stride2(DR["s1"], 256, 2, _dt),
        f"stride2_c4_s2_c512_{_dt}": Stride2(D4["s2"], 512, 1, _dt),
        f"stride2_small_s3_c1024_{_dt}": Stride2(DS["s3"], 1024, 1, _dt),
        f"pack_64x256x1_{_dt}": Pack(64, 256, 1, _dt),
        f"pack_256x64x3_{_dt}": Pack(256, 64, 3, _dt),
        f"pack_120x256x1_{_dt}": Pack(120, 256, 1, _dt),
        f"pack_256x256x3_fwd_only_{_dt}": Pack(256, 256, 3, _dt, bwd=False),
        f"stem_s1_vgg32_{_dt}": StemS1((32, 32, 32), 1, _dt),
        f"stem_s1_odd_n2_{_dt}": StemS1((21, 18, 14), 2, _dt),
        f"pool2_vgg_odd_n2_{_dt}": Pool2((5, 7, 3), 64, 2, _dt),
        f"loss_obb_{_dt}": Loss(True, _dt),
        f"loss_aabb_{_dt}": Loss(False, _dt),
        f"loss_obb_theta_edges_{_dt}": Loss(True, _dt, (64,), (64,), theta=(0.0, math.pi / 2, -math.pi / 2, math.pi / 4)),
        f"loss_background_{_dt}": Loss(True, _dt, (0,), (256,)),                 # a scene with no positive
        f"loss_256_samples_w_reg0_{_dt}": Loss(False, _dt, (128,), (128,), w_reg=0.0),
        f"loss_batch3_{_dt}": Loss(True, _dt, (40, 0, 128), (216, 256, 128)),
    })
    for _c, _d in zip((64, 128, 256, 512), VGG):
        ROWS[f"pool2_vgg_c{_c}_{_dt}"] = Pool2(_d, _c, 1, _dt)
ROWS.update({
    "opt_3steps_step2_clipped": Opt(1_000_003, steps=(1, 2, 3), grad_std=(1e-5, 1e-2, 1e-5)),
    "opt_frozen_head_obb_fp16": Opt(HEAD_N[True], HEAD_LO, 1 / 1024, steps=(1, 2), grad_std=(1e-2, 1e-4)),
    "opt_frozen_head_aabb": Opt(HEAD_N[False], HEAD_LO, steps=(7,), grad_std=(1e-3,), warm=True),
    "opt_unaligned_offset1": Opt(1_000_003, 1, 1 / 1024, steps=(2,), grad_std=(1e-2,), warm=True),
    "opt_n100_fewer_than_blocks": Opt(100, steps=(1,), grad_std=(1.0,)),
    "opt_max_norm0": Opt(65_537, max_norm=0.0, steps=(1, 2), grad_std=(1.0, 1e-3)),
    "opt_late_step": Opt(262_147, steps=(10_000,), grad_std=(1e-4,), warm=True),
    "opt_not_clipped_warm": Opt(262_147, max_norm=10.0, steps=(5,), grad_std=(1e-3,), warm=True),
})


# ------------------------------------------------------------------------------------------------ bounds (shared with the CPU controls)
def bn_chain(rows, c):
    blocks = min(rows, RED_BLOCKS)
    per = -(-rows // blocks)
    lanes = max(256 // (c // 8), 1)
    return -(-per // lanes) + lanes


def bn_stats_bounds(ref, rows, c, eps=EPS, momentum=0.1):
    """Per-channel bounds of mean, rstd, var and the running statistics (dict of float64 tensors)."""
    k = bn_chain(rows, c) + 2
    d_mean = k * E * ref["e_abs"]
    d_var = 3 * k * E * ref["e_sq"]
    out = dict(mean=d_mean + E * ref["mean"].abs(), var=d_var + E * ref["var"], rstd=ref["rstd"] * (0.5 * d_var / (ref["var"] + eps) + 2 * E))
    if "running_mean" in ref:
        out["running_mean"] = momentum * d_mean + E * ref["running_mean"].abs() + 1e-30
        out["running_var"] = momentum * d_var * rows / max(rows - 1, 1) + E * ref["running_var"].abs()
    return out


def act_bound(ref, scale, dtype, terms):
    return HALF_ULP[dtype] * ref.abs() + terms * E * scale + E


def bn_sum_bounds(ref, rows, c):
    k = bn_chain(rows, c)
    return ((k + 4) * E * ref["mag_dgamma"] + E * ref["dgamma"].abs() + 1e-30, (k + 1) * E * ref["mag_dbeta"] + E * ref["dbeta"].abs() + 1e-30)


def target_bound(tmag):
    return 16 * E * tmag


def loss_bounds(ref, targets, tmag, pred, dtype, norm, w_obj, w_reg, grad_scale):
    """(dlogit bound, ddelta bound, l_obj bound, l_reg bound) of one nrpn_rpn_loss call."""
    u = HALF_ULP[dtype]
    k, kr = w_obj * grad_scale / norm, w_reg * grad_scale / norm
    dd = target_bound(tmag) + 2 * E * (pred.double().abs() + targets.abs())
    b_logit = u * ref["dlogit"].abs() + 8 * E * k + E
    b_delta = u * ref["ddelta"].abs() + 9 * kr * dd + E
    b_obj = 8 * E * float(ref["mag_obj"].sum()) / norm + 2 * E * abs(ref["l_obj"])
    b_reg = (float(dd.sum()) + 4 * E * float(ref["d"].abs().sum())) / norm + 2 * E * abs(ref["l_reg"])
    return b_logit, b_delta, b_obj, b_reg


def f32(v):
    return float(np.float32(v))


def adamw_bounds(p, g, m, v, ref, norm, max_norm, inv_scale, lr, beta1, beta2, eps, step):
    """Bounds of (p, m, v) after one nrpn_adamw_step; ref = reference_adamw64(...) on the same fp32 operands."""
    p1, m1, v1, u = ref
    coef = inv_scale * (min(max_norm / (float(norm) + 1e-6), 1.0) if max_norm > 0 else 1.0)
    gi = g.double().abs() * coef
    rel_g = 6 * E
    b1t, b2t = beta1 ** step, beta2 ** step
    rel_bc1 = E * (b1t / (1 - b1t) + 1)
    rel_bc2s = 0.5 * E * (b2t / (1 - b2t) + 1) + E
    b_m = 3 * E * (beta1 * m.double().abs() + (1 - beta1) * gi) + (1 - beta1) * rel_g * gi + E * m1.abs()
    rel_v = 3 * E + 2 * rel_g
    b_v = (rel_v + E) * v1
    rel_den = 0.5 * rel_v + rel_bc2s + 3 * E
    k = lr / (1 - b1t) / (torch.sqrt(v1 / (1 - b2t)) + eps)     # what an error of m reaches p multiplied by
    b_p = 4 * E * (p.double().abs() + p1.abs()) + u * (rel_bc1 + rel_den + 4 * E) + k * b_m + 1e-30
    return b_p, b_m + 1e-30, b_v + 1e-30


# ------------------------------------------------------------------------------------------------ helpers
def _gen(name, device="cuda"):
    return torch.Generator(device=device).manual_seed(zlib.crc32(name.encode()) % 100000)


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _nan_buffer(shape, dtype, fill=None):
    numel = math.prod(shape)
    buf = torch.full((numel + 2 * GUARD,), float("nan"), dtype=dtype, device="cuda")
    view = buf[GUARD: GUARD + numel].view(shape)
    if fill is not None:
        view.copy_(fill)
    return buf, view


def _ibits(t):
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _guards_intact(buf, tag):
    bits, nan = _ibits(buf), _ibits(torch.full((1,), float("nan"), dtype=buf.dtype, device="cuda"))
    assert bool((bits[:GUARD] == nan).all()) and bool((bits[-GUARD:] == nan).all()), f"{tag}: written outside the output"


def _finite(t, tag):
    assert bool(torch.isfinite(t).all()), f"{tag}: {int((~torch.isfinite(t)).sum())} outputs unwritten or not finite"


def _within(got, ref, bound, tag):
    err = (got.double() - ref).abs()
    ratio = err / bound
    at = int(ratio.argmax())
    worst = float(ratio.reshape(-1)[at])
    assert bool((err <= bound).all()), (f"{tag}: {int((err > bound).sum())} of {err.numel()} out of bound; worst err/bound {worst:.3g}: "
                                       f"got {float(got.reshape(-1)[at]):.8g} ref {float(ref.reshape(-1)[at]):.8g} bound {float(bound.reshape(-1)[at]):.3g}")
    return worst


def _same_bits(got, want, tag):
    diff = _ibits(got) != _ibits(want)
    assert not bool(diff.any()), f"{tag}: {int(diff.sum())} of {got.numel()} elements differ"


def _check(rc, what):
    from nerf_rpn_b200._lib import check
    check(rc, what)


# ------------------------------------------------------------------------------------------------ rows
def bn_operands(row, name, device):
    """y, res (None unless residual), gamma, beta, dout, running mean and variance of a BN row (CPU or GPU)."""
    dt, g, rows, c = DTYPE[row.dtype], _gen(name, device), row.rows, row.c
    y = (torch.randn(rows, c, device=device, generator=g) * row.std + row.mean).to(dt)
    res = torch.randn(rows, c, device=device, generator=g).to(dt) if row.kind == "residual" else None
    gamma = torch.rand(c, device=device, generator=g) + 0.5
    beta = torch.randn(c, device=device, generator=g) * 0.2
    dout = (torch.randn(rows, c, device=device, generator=g) * 0.01).to(dt)
    if row.running:
        rm0, rv0 = torch.randn(c, device=device, generator=g) * 0.5, torch.rand(c, device=device, generator=g) + 0.5
    else:
        rm0, rv0 = torch.zeros(c, device=device), torch.ones(c, device=device)
    return y, res, gamma, beta, dout, rm0, rv0


def _run_bn(L, row, name):
    dt, u = DTYPE[row.dtype], HALF_ULP[DTYPE[row.dtype]]
    f16 = int(dt == torch.float16)
    rows, c = row.rows, row.c
    relu, has_res = row.kind != "plain", row.kind == "residual"
    y, res, gamma, beta, dout, rm0, rv0 = bn_operands(row, name, "cuda")
    ws = torch.empty(L.nrpn_chan_reduce_workspace_bytes(c), dtype=torch.uint8, device="cuda")
    sbuf, stats = _nan_buffer((3 * c,), torch.float32)
    rmb, rm = _nan_buffer((c,), torch.float32, rm0)
    rvb, rv = _nan_buffer((c,), torch.float32, rv0)
    _check(L.nrpn_bn_stats(_p(y), rows, c, f16, EPS, _p(stats), _p(rm), _p(rv), 0.1, _p(ws), ws.numel(), _s()), "bn_stats")
    obuf, out = _nan_buffer((rows, c), dt)
    _check(L.nrpn_bn_apply(_p(y), _p(res), _p(out), rows, c, _p(stats), _p(gamma), _p(beta), int(relu), f16, _s()), "bn_apply")
    sumbuf, sums = _nan_buffer((2 * c,), torch.float32)
    dybuf, dy = _nan_buffer((rows, c), dt)
    drbuf, dres = _nan_buffer((rows, c), dt) if has_res else (None, None)
    _check(L.nrpn_bn_backward(_p(dout), _p(out if relu else None), _p(y), _p(dy), _p(dres), rows, c, _p(stats), _p(gamma), _p(sums),
                              int(relu), f16, _p(ws), ws.numel(), _s()), "bn_backward")
    torch.cuda.synchronize()
    for b, t in ((sbuf, "stats"), (rmb, "running_mean"), (rvb, "running_var"), (obuf, "out"), (sumbuf, "sums"), (dybuf, "dy"), (drbuf, "dres")):
        if b is not None:
            _guards_intact(b, f"{name} {t}")
            _finite(b[GUARD:-GUARD], f"{name} {t}")
    # statistics against the exact float64 ones
    ref = reference_bn_stats64(y, f32(EPS), rm0, rv0, f32(0.1))
    bnd = bn_stats_bounds(ref, rows, c)
    worst = max(_within(stats[:c], ref["mean"], bnd["mean"], f"{name} mean"), _within(stats[c:2 * c], ref["rstd"], bnd["rstd"], f"{name} rstd"),
                _within(stats[2 * c:], ref["var"], bnd["var"], f"{name} var"),
                _within(rm, ref["running_mean"], bnd["running_mean"], f"{name} running_mean"),
                _within(rv, ref["running_var"], bnd["running_var"], f"{name} running_var"))
    mean, rstd = stats[:c], stats[c:2 * c]
    # apply, backward sums, then dy / dres on the statistics and sums the kernels read, CHUNK rows at a time
    sg = torch.zeros(c, dtype=torch.float64, device="cuda")
    sb, mg, mb = torch.zeros_like(sg), torch.zeros_like(sg), torch.zeros_like(sg)
    for r0 in range(0, rows, CHUNK):
        sl = slice(r0, r0 + CHUNK)
        r_out, scale = reference_bn_apply64(y[sl], None if res is None else res[sl], mean, rstd, gamma, beta, relu)
        worst = max(worst, _within(out[sl], r_out, act_bound(r_out, scale, dt, 8), f"{name} out"))
        rb = reference_bn_backward64(dout[sl], out[sl], y[sl], mean, rstd, gamma, relu, sums=(sums[:c], sums[c:]), rows=rows)
        sg += rb["dgamma"]; sb += rb["dbeta"]; mg += rb["mag_dgamma"]; mb += rb["mag_dbeta"]
        worst = max(worst, _within(dy[sl], rb["dy"], act_bound(rb["dy"], rb["mag_dy"], dt, 10), f"{name} dy"))
        if has_res:
            worst = max(worst, _within(dres[sl], rb["dres"], u * rb["dres"].abs() + E, f"{name} dres"))
    b_g, b_b = bn_sum_bounds(dict(dgamma=sg, dbeta=sb, mag_dgamma=mg, mag_dbeta=mb), rows, c)
    worst = max(worst, _within(sums[:c], sg, b_g, f"{name} dgamma"), _within(sums[c:], sb, b_b, f"{name} dbeta"))
    return worst


def _run_pool(L, row, name):
    dt = DTYPE[row.dtype]
    f16 = int(dt == torch.float16)
    g = _gen(name)
    x = torch.randn(row.n, *row.dims, row.c, device="cuda", generator=g)
    x = (x - 2.0).clamp_min(0).to(dt) if row.post_relu else x.to(dt)
    od = tuple((d - 1) // 2 + 1 for d in row.dims)
    want, code = reference_maxpool3_argmax(x)
    obuf, out = _nan_buffer((row.n, *od, row.c), dt)
    ibuf = torch.full((math.prod(out.shape) + 2 * GUARD,), 0xEE, dtype=torch.uint8, device="cuda")     # 0xEE is no window position
    idx = ibuf[GUARD:-GUARD].view(out.shape)
    _check(L.nrpn_maxpool3d_k3s2_argmax(_p(x), row.n, *row.dims, row.c, _p(out), _p(idx), f16, _s()), "maxpool_argmax")
    pbuf, plain = _nan_buffer((row.n, *od, row.c), dt)
    _check(L.nrpn_maxpool3d_k3s2(_p(x), row.n, *row.dims, row.c, _p(plain), f16, _s()), "maxpool")
    dyo = torch.randn(row.n, *od, row.c, device="cuda", generator=g).to(dt)
    dbuf, dx = _nan_buffer(tuple(x.shape), dt)
    _check(L.nrpn_maxpool3d_k3s2_backward(_p(dyo), _p(idx), row.n, *row.dims, row.c, _p(dx), f16, _s()), "maxpool_backward")
    torch.cuda.synchronize()
    for b, t in ((obuf, "out"), (pbuf, "plain out"), (dbuf, "dx")):
        _guards_intact(b, f"{name} {t}")
    assert bool((ibuf[:GUARD] == 0xEE).all()) and bool((ibuf[-GUARD:] == 0xEE).all()), f"{name}: argmax written outside"
    _same_bits(out, want, f"{name} out")
    _same_bits(plain, want, f"{name} plain out")
    assert torch.equal(idx, code), f"{name}: {int((idx != code).sum())} argmax codes differ"
    if row.post_relu:
        assert float((want == 0).float().mean()) > 0.05, f"{name}: too few all-zero windows to test the tie rule"
    _finite(dx, f"{name} dx")
    ref, mag = reference_maxpool3_backward64(dyo, code, row.dims)
    return _within(dx, ref, act_bound(ref, mag, dt, 8), f"{name} dx")


def _run_pool2(L, row, name):
    dt = DTYPE[row.dtype]
    x = torch.randn(row.n, *row.dims, row.c, device="cuda", generator=_gen(name)).to(dt)
    want = reference_maxpool2_ceil(x)
    buf, out = _nan_buffer(tuple(want.shape), dt)
    _check(L.nrpn_maxpool3d_k2s2_ceil(_p(x), row.n, *row.dims, row.c, _p(out), int(dt == torch.float16), _s()), "maxpool_k2s2_ceil")
    torch.cuda.synchronize()
    _guards_intact(buf, name)
    _same_bits(out, want, name)
    return 0.0


def _run_up(L, row, name):
    dt = DTYPE[row.dtype]
    g = _gen(name)
    df = torch.randn(row.n, *row.fine, row.c, device="cuda", generator=g).to(dt)
    dc0 = torch.randn(row.n, *row.coarse, row.c, device="cuda", generator=g).to(dt)
    buf, dc = _nan_buffer(tuple(dc0.shape), dt, dc0)
    _check(L.nrpn_upsample_nearest_backward(_p(df), row.n, *row.fine, *row.coarse, row.c, _p(dc), int(dt == torch.float16), _s()), "upsample_backward")
    torch.cuda.synchronize()
    _guards_intact(buf, name)
    _finite(dc, name)
    ref, mag, terms = reference_upsample_backward64(df, dc0)
    return _within(dc, ref, act_bound(ref, mag, dt, terms + 1), name)


def _run_stride2(L, row, name):
    dt = DTYPE[row.dtype]
    x = torch.randn(row.n, *row.dims, row.c, device="cuda", generator=_gen(name)).to(dt)
    od = tuple((d + 1) // 2 for d in row.dims)
    gbuf, xs = _nan_buffer((row.n, *od, row.c), dt)
    _check(L.nrpn_stride2(_p(x), _p(xs), row.n, *row.dims, row.c, 0, _s()), "stride2 gather")
    sbuf, back = _nan_buffer(tuple(x.shape), dt)
    _check(L.nrpn_stride2(_p(xs), _p(back), row.n, *row.dims, row.c, 1, _s()), "stride2 scatter")
    a0 = x.clone()
    abuf, a = _nan_buffer(tuple(x.shape), dt, a0)
    b = torch.randn(x.shape, device="cuda", generator=_gen(name + "b")).to(dt)
    _check(L.nrpn_add_inplace(_p(a), _p(b), a.numel(), int(dt == torch.float16), _s()), "add_inplace")
    torch.cuda.synchronize()
    for bf, t in ((gbuf, "gather"), (sbuf, "scatter"), (abuf, "add")):
        _guards_intact(bf, f"{name} {t}")
    _same_bits(xs, x[:, ::2, ::2, ::2].contiguous(), f"{name} gather")
    want = torch.zeros_like(x)
    want[:, ::2, ::2, ::2] = xs
    _same_bits(back, want, f"{name} scatter")
    ref = a0.double() + b.double()
    return _within(a, ref, act_bound(ref, ref.abs(), dt, 1), f"{name} add")


def _run_pack(L, row, name):
    from nerf_rpn_b200 import packing
    dt = DTYPE[row.dtype]
    w = torch.randn(row.cout, row.cin, row.k, row.k, row.k, device="cuda", generator=_gen(name))
    fwd_ref, _ = packing.pack_conv_weight(w.cpu(), dtype=dt)
    bwd_ref, _ = packing.pack_conv_weight_dgrad(w.cpu(), dtype=dt)
    fbuf, fwd = _nan_buffer(tuple(fwd_ref.shape), dt, torch.zeros(fwd_ref.shape, dtype=dt, device="cuda"))
    bbuf, bwd = _nan_buffer(tuple(bwd_ref.shape), dt, torch.zeros(bwd_ref.shape, dtype=dt, device="cuda"))
    _check(L.nrpn_pack_weights(_p(w), row.cout, row.cin, row.k ** 3, _p(fwd), fwd.shape[1], fwd.shape[2], _p(bwd if row.bwd else None),
                               bwd.shape[1], bwd.shape[2], int(dt == torch.float16), _s()), "pack_weights")
    torch.cuda.synchronize()
    _guards_intact(fbuf, name); _guards_intact(bbuf, name)
    _same_bits(fwd.cpu(), fwd_ref, f"{name} fwd")
    _same_bits(bwd.cpu(), bwd_ref if row.bwd else torch.zeros_like(bwd_ref), f"{name} bwd")
    return 0.0


def _run_stem_s1(L, row, name):
    dt = DTYPE[row.dtype]
    grid = torch.randn(row.n, 4, *row.dims, device="cuda", generator=_gen(name)) * 3
    want = emulate_pack_stem_s1(grid.double()).to(dt)
    buf, out = _nan_buffer(tuple(want.shape), dt)
    _check(L.nrpn_pack_stem_input_s1(_p(grid), row.n, *row.dims, _p(out), int(dt == torch.float16), _s()), "pack_stem_input_s1")
    torch.cuda.synchronize()
    _guards_intact(buf, name)
    _same_bits(out, want, name)
    return 0.0


LOSS_DIMS, LOSS_FD = (32, 48, 40), ((8, 12, 10), (4, 6, 5), (2, 3, 3), (1, 2, 2))


def loss_setup(row, name, device):
    """Predictor rows, sampled anchor indices and their gt boxes for each call of a Loss row (CPU or GPU)."""
    from nerf_rpn_b200.model.anchor import AnchorGenerator3D
    from oracle import ref_gpu
    cells = AnchorGenerator3D(ref_gpu.ANCHOR_SIZES, ref_gpu.ASPECT).cell_anchors_np()
    strides = [tuple(LOSS_DIMS[k] // d[k] for k in range(3)) for d in LOSS_FD]
    A, code = 13, 8 if row.rotated else 6
    total = sum(_vol(d) for d in LOSS_FD) * A
    g = _gen(name, device)
    calls = []
    for n_pos, n_neg in zip(row.n_pos, row.n_neg):
        preds = []
        for d in LOSS_FD:
            p = torch.full((_vol(d), 128), float("nan"), device=device)            # pad columns past A (1 + code) are never read
            p[:, :A * (1 + code)] = torch.randn(_vol(d), A * (1 + code), device=device, generator=g) * 0.5
            preds.append(p)
        perm = torch.randperm(total, device=device, generator=g)
        pos, neg = perm[:n_pos].contiguous(), perm[n_pos:n_pos + n_neg].contiguous()
        _, _, _, an = rpn_anchors_f32(pos, LOSS_FD, strides, cells, A)
        ctr, size = (an[:, :3] + an[:, 3:]) / 2, an[:, 3:] - an[:, :3]
        jitter = torch.randn(n_pos, 3, device=device, generator=g) * 0.1 * size
        scale = torch.exp(torch.randn(n_pos, 3, device=device, generator=g) * 0.2)
        if row.rotated:
            if row.theta is None:
                th = (torch.rand(n_pos, 1, device=device, generator=g) - 0.5) * math.pi
            else:
                th = torch.tensor(row.theta, device=device).repeat(-(-n_pos // len(row.theta)))[:n_pos, None].float()
            gt = torch.cat([ctr + jitter, size * scale, th], 1).contiguous()
        else:
            c2, s2 = ctr + jitter, size * scale
            gt = torch.cat([c2 - s2 / 2, c2 + s2 / 2], 1).contiguous()
        calls.append((preds, pos, neg, gt))
    return calls, cells, strides, A, code


def _run_loss(L, row, name):
    from nerf_rpn_b200 import ops
    from oracle import loss_oracle as lo
    dt = DTYPE[row.dtype]
    calls, cells, strides, A, code = loss_setup(row, name, "cuda")
    norm = float(sum(row.n_pos) + sum(row.n_neg))
    w_obj, grad_scale = 1.0, 256.0
    lbuf, losses = _nan_buffer((2,), torch.float32, torch.tensor([0.25, 0.5], device="cuda"))
    want_obj, want_reg, b_obj, b_reg, worst = 0.25, 0.5, 0.0, 0.0, 0.0
    for ci, (preds, pos, neg, gt) in enumerate(calls):
        tag = f"{name} call {ci}"
        dbufs = [_nan_buffer(tuple(p.shape), dt) for p in preds]
        tbuf, tout = _nan_buffer((pos.numel(), code), torch.float32)
        desc = ops.make_rpn_desc(preds, LOSS_FD, strides, cells, A, row.rotated, 1, 1, 0.5, 0.0, 1e-3, LOSS_DIMS)
        arr = (ctypes.c_void_p * 4)(*[v.data_ptr() for _, v in dbufs])
        _check(L.nrpn_rpn_loss(ctypes.byref(desc), arr, _p(pos), pos.numel(), _p(neg), neg.numel(), _p(gt), norm, w_obj, row.w_reg, grad_scale,
                               _p(losses), _p(tout), int(dt == torch.float16), _s()), "rpn_loss")
        torch.cuda.synchronize()
        samp = torch.cat([pos, neg])
        lvl, vox, a, an = rpn_anchors_f32(samp, LOSS_FD, strides, cells, A)
        logits = torch.stack([preds[int(l)][int(v), int(aa)] for l, v, aa in zip(lvl.tolist(), vox.tolist(), a.tolist())]) if samp.numel() else torch.zeros(0, device="cuda")
        npos = pos.numel()
        cols = (A + a[:npos] * code).view(-1, 1) + torch.arange(code, device="cuda").view(1, -1)
        prow = torch.zeros((npos, code), device="cuda")
        for l in range(4):
            m = lvl[:npos] == l
            if bool(m.any()):
                prow[m] = preds[l][vox[:npos][m].view(-1, 1), cols[m]]
        t, tmag = encode_targets64(an[:npos], gt, row.rotated)
        ref = reference_rpn_loss64(prow, logits, npos, t, norm, w_obj, row.w_reg, grad_scale)
        bl, bd, bo, br = loss_bounds(ref, t, tmag, prow, dt, norm, w_obj, row.w_reg, grad_scale)
        want_obj += ref["l_obj"]; want_reg += ref["l_reg"]; b_obj += bo + E * abs(want_obj); b_reg += br + E * abs(want_reg)
        _guards_intact(tbuf, f"{tag} targets")
        if npos:
            _finite(tout, f"{tag} targets")
            worst = max(worst, _within(tout, t, target_bound(tmag), f"{tag} targets"))
            an_np, gt_np = an[:npos].cpu().numpy(), gt.cpu().numpy()
            enc = lo.encode_obb_midpoint(an_np, gt_np) if row.rotated else lo.encode_aabb(gt_np, an_np)
            assert np.allclose(tout.cpu().numpy(), enc, rtol=2e-5, atol=2e-6), f"{tag}: targets vs oracle/loss_oracle.py {np.abs(tout.cpu().numpy() - enc).max()}"
        # every element of the predictor gradient: sampled logits and positive deltas within bound, everything else untouched
        written = [torch.zeros(p.shape, dtype=torch.bool, device="cuda") for p in preds]
        for l in range(4):
            m = lvl == l
            if bool(m.any()):
                got = dbufs[l][1][vox[m], a[m]]
                _finite(got, f"{tag} dlogit")
                worst = max(worst, _within(got, ref["dlogit"][m], bl[m], f"{tag} dlogit"))
                written[l][vox[m], a[m]] = True
            mp = lvl[:npos] == l
            if bool(mp.any()):
                got = dbufs[l][1][vox[:npos][mp].view(-1, 1), cols[mp]]
                _finite(got, f"{tag} ddelta")
                worst = max(worst, _within(got, ref["ddelta"][mp], bd[mp], f"{tag} ddelta"))
                written[l][vox[:npos][mp].view(-1, 1), cols[mp]] = True
        for l, (buf, view) in enumerate(dbufs):
            _guards_intact(buf, f"{tag} dpred[{l}]")
            assert bool(torch.isnan(view[~written[l]]).all()), f"{tag}: dpred[{l}] written away from the sampled anchors"
    torch.cuda.synchronize()
    _guards_intact(lbuf, f"{name} losses")
    worst = max(worst, abs(float(losses[0]) - want_obj) / b_obj, abs(float(losses[1]) - want_reg) / b_reg)
    assert abs(float(losses[0]) - want_obj) <= b_obj and abs(float(losses[1]) - want_reg) <= b_reg, \
        (f"{name} losses", losses.tolist(), want_obj, want_reg, b_obj, b_reg)
    return worst


OPT_HP = (3e-4, 0.9, 0.999, 1e-8, 0.01)           # lr, beta1, beta2, eps, weight decay


def _run_opt(L, row, name):
    g = _gen(name)
    lr, b1, b2, eps, wd = OPT_HP
    total = row.offset + row.n
    def buf(fill):
        b, v = _nan_buffer((total,), torch.float32)
        v[row.offset:] = fill
        return b, v
    pb, pf = buf(torch.randn(row.n, device="cuda", generator=g))
    mb, mf = buf(torch.randn(row.n, device="cuda", generator=g) * 1e-3 if row.warm else torch.zeros(row.n, device="cuda"))
    vb, vf = buf(torch.rand(row.n, device="cuda", generator=g) * 1e-6 if row.warm else torch.zeros(row.n, device="cuda"))
    gb, gf = _nan_buffer((total,), torch.float32)
    nb, norm = _nan_buffer((1,), torch.float32)
    ws = torch.empty(L.nrpn_grad_norm_workspace_bytes(), dtype=torch.uint8, device="cuda")
    worst = 0.0
    for step, std in zip(row.steps, row.grad_std):
        gf[row.offset:] = torch.randn(row.n, device="cuda", generator=g) * (std / row.inv_scale)
        p0, m0, v0 = (t[row.offset:].clone() for t in (pf, mf, vf))
        gr = gf[row.offset:]
        ptrs = [ctypes.c_void_p(t.data_ptr() + 4 * row.offset) for t in (pf, gf, mf, vf)]
        _check(L.nrpn_grad_norm(ptrs[1], row.n, row.inv_scale, _p(norm), _p(ws), ws.numel(), _s()), "grad_norm")
        _check(L.nrpn_adamw_step(ptrs[0], ptrs[1], ptrs[2], ptrs[3], row.n, _p(norm), row.max_norm, row.inv_scale, lr, b1, b2, eps, wd, step, _s()),
               "adamw_step")
        torch.cuda.synchronize()
        tag = f"{name} step {step}"
        want = reference_grad_norm64(gr, row.inv_scale)
        worst = max(worst, abs(float(norm) - want) / (2.0 ** -22 * want))
        assert abs(float(norm) - want) <= 2.0 ** -22 * want, (tag, float(norm), want)
        hp = (f32(row.max_norm), f32(row.inv_scale), f32(lr), f32(b1), f32(b2), f32(eps), f32(wd))
        ref = reference_adamw64(p0, gr, m0, v0, float(norm), hp[0], hp[1], hp[2], hp[3], hp[4], hp[5], hp[6], step)
        bp, bm, bv = adamw_bounds(p0, gr, m0, v0, ref, float(norm), hp[0], hp[1], hp[2], hp[3], hp[4], hp[5], step)
        _guards_intact(nb, f"{tag} norm")
        for b, t in ((pb, "p"), (mb, "m"), (vb, "v"), (gb, "g")):
            _guards_intact(b, f"{tag} {t}")
            assert bool(torch.isnan(b[GUARD:GUARD + row.offset]).all()), f"{tag}: {t} written before its range"
        worst = max(worst, _within(pf[row.offset:], ref[0], bp, f"{tag} p"), _within(mf[row.offset:], ref[1], bm, f"{tag} m"),
                    _within(vf[row.offset:], ref[2], bv, f"{tag} v"))
    return worst


RUN = {BN: _run_bn, Pool: _run_pool, Pool2: _run_pool2, Up: _run_up, Stride2: _run_stride2, Pack: _run_pack, StemS1: _run_stem_s1,
       Loss: _run_loss, Opt: _run_opt}


@pytest.fixture(scope="module")
def L():
    assert torch.cuda.is_available()
    from nerf_rpn_b200._lib import lib
    return lib()


@pytest.mark.parametrize("name", list(ROWS))
def test_kernel_row(L, name):
    row = ROWS[name]
    worst = RUN[type(row)](L, row, name)
    exact = isinstance(row, (Pool2, Pack, StemS1))
    print(f"\n[bandwidth kernel] {name:40s} worst err/bound {worst:.3g}" + ("  (bit-exact)" if exact else ""))


# ------------------------------------------------------------------------------------------------ coverage
def row_keys(row):
    """The (entry point, channels, flags, dtype) launch combinations a row exercises."""
    dt = row.dtype if hasattr(row, "dtype") else None
    if isinstance(row, BN):
        relu, res = row.kind != "plain", row.kind == "residual"
        return {("bn_stats", row.c, 1, dt), ("bn_apply", row.c, (relu, res), dt), ("bn_backward", row.c, (relu, res), dt)}
    if isinstance(row, Pool):
        return {("maxpool3d_k3s2_argmax", row.c, 0, dt), ("maxpool3d_k3s2_backward", row.c, 0, dt), ("maxpool3d_k3s2", row.c, 0, dt)}
    if isinstance(row, Pool2):
        return {("maxpool3d_k2s2_ceil", row.c, 0, dt)}
    if isinstance(row, Up):
        return {("upsample_nearest_backward", row.c, 0, dt)}
    if isinstance(row, Stride2):
        return {("stride2", row.c, 0, None), ("stride2", row.c, 1, None), ("add_inplace", 0, 0, dt)}
    if isinstance(row, Pack):
        return {("pack_weights", 0, int(row.bwd), dt)}
    if isinstance(row, StemS1):
        return {("pack_stem_input_s1", 0, 0, dt)}
    if isinstance(row, Loss):
        return {("rpn_loss", 0, int(row.rotated), dt)}
    return {("grad_norm", 0, 0, None), ("adamw_step", 0, int(row.max_norm > 0), None)}


def _nonnull(v):
    return (v.value is not None) if isinstance(v, ctypes.c_void_p) else bool(v)


def _dt(f16):
    return "fp16" if f16 else "bf16"


RECORDERS = {
    "nrpn_bn_stats": lambda a: ("bn_stats", a[2], int(_nonnull(a[6])), _dt(a[3])),
    "nrpn_bn_apply": lambda a: ("bn_apply", a[4], (bool(a[8]), _nonnull(a[1])), _dt(a[9])),
    "nrpn_bn_backward": lambda a: ("bn_backward", a[6], (bool(a[10]), _nonnull(a[4])), _dt(a[11])),
    "nrpn_maxpool3d_k3s2_argmax": lambda a: ("maxpool3d_k3s2_argmax", a[5], 0, _dt(a[8])),
    "nrpn_maxpool3d_k3s2_backward": lambda a: ("maxpool3d_k3s2_backward", a[6], 0, _dt(a[8])),
    "nrpn_maxpool3d_k3s2": lambda a: ("maxpool3d_k3s2", a[5], 0, _dt(a[7])),
    "nrpn_maxpool3d_k2s2_ceil": lambda a: ("maxpool3d_k2s2_ceil", a[5], 0, _dt(a[7])),
    "nrpn_upsample_nearest_backward": lambda a: ("upsample_nearest_backward", a[8], 0, _dt(a[10])),
    "nrpn_stride2": lambda a: ("stride2", a[6], int(bool(a[7])), None),
    "nrpn_add_inplace": lambda a: ("add_inplace", 0, 0, _dt(a[3])),
    "nrpn_rpn_loss": lambda a: ("rpn_loss", 0, int(a[0]._obj.rotated), _dt(a[13])),
    "nrpn_pack_weights": lambda a: ("pack_weights", 0, int(_nonnull(a[7])), _dt(a[10])),
    "nrpn_pack_stem_input_s1": lambda a: ("pack_stem_input_s1", 0, 0, _dt(a[6])),
    "nrpn_grad_norm": lambda a: ("grad_norm", 0, 0, None),
    "nrpn_adamw_step": lambda a: ("adamw_step", 0, int(a[6] > 0), None),
}


def test_table_covers_every_path(L, monkeypatch):
    """Every launch combination of one eager full and one eager frozen training step of the (2,1,1,1) engine in each precision, a
    fp16_w2 ResNet inference forward and a VGG small-grid inference forward has a row."""
    from nerf_rpn_b200.model.anchor import AnchorGenerator3D, RPNHead
    from nerf_rpn_b200.model.feature_extractor import VGG_FPN
    from nerf_rpn_b200.model.nerf_rpn import NeRFRegionProposalNetwork
    from nerf_rpn_b200.train import RPNTrainEngine
    from oracle import ref_gpu
    from tests.test_gpu_train import _planted
    from tests.test_gpu_train_ragged import _model
    seen = set()
    for entry, key in RECORDERS.items():
        fn = getattr(L, entry)

        def wrapped(*args, _fn=fn, _key=key):
            seen.add(_key(args))
            return _fn(*args)
        monkeypatch.setattr(L, entry, wrapped)
    dims = (64, 96, 80)
    for precision in ("bf16", "fp16"):
        for frozen in (False, True):
            grid, gt = _planted(dims, 12, 11, True)
            eng = RPNTrainEngine(_model((2, 1, 1, 1), True), precision=precision, seed=7, freeze_backbone=frozen, reg_loss_weight=5.0)
            eng.forward_backward(grid.cuda()[None], [gt.cuda()])
            eng.optimizer_step()
            torch.cuda.synchronize()
            del eng
    model = _model((3, 4, 6, 3), False).eval()                           # the inference engine runs the ResNet50 backbone only
    model.precision = model.backbone.precision = "fp16_w2"
    with torch.no_grad():
        model([torch.rand(4, *dims, device="cuda")])
    torch.manual_seed(0)
    vgg = NeRFRegionProposalNetwork(VGG_FPN("EF", 4, True, 32), AnchorGenerator3D(ref_gpu.ANCHOR_SIZES, ref_gpu.ASPECT), RPNHead(256, 13, 4),
                                    rpn_pre_nms_top_n_test=100, rpn_post_nms_top_n_test=100).cuda().eval()
    vgg.precision = vgg.backbone.precision = "fp16_w2"
    with torch.no_grad():
        vgg([torch.rand(4, 32, 32, 32, device="cuda")])
    torch.cuda.synchronize()
    covered = set().union(*(row_keys(r) for r in ROWS.values()))
    print(f"\n{len(seen)} launch combinations recorded")
    assert seen, "nothing recorded"
    missing = sorted(seen - covered, key=repr)
    assert not missing, f"launch combinations without a row: {missing}"

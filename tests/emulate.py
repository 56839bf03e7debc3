"""Pure-torch statement of what nrpn_conv3d_fprop / nrpn_conv3d_wgrad / nrpn_pack_stem_input, the Swin-3D / GroupNorm kernels and the
training step's bandwidth kernels compute (TEST helper, CPU or GPU).  Used to check the host-side packing logic without a GPU and as
the fp32 / float64 references for the CUDA kernels."""
import math

import torch
import torch.nn.functional as F


def emulate_pack_stem(grid: torch.Tensor) -> torch.Tensor:
    """(N,4,X,Y,Z) fp32 -> (N,X2,Y2,Z2+1,64) fp32 with the layout of csrc/pointwise.cu:pack_stem_kernel."""
    n, c, X, Y, Z = grid.shape
    X2, Y2, Z2 = (X + 1) // 2, (Y + 1) // 2, (Z + 1) // 2
    g = F.pad(grid, (0, 2 * Z2 - Z, 0, 2 * Y2 - Y, 0, 2 * X2 - X))
    # s2d block: channel = ((rx*2+ry)*2+rz)*4 + c
    b = g.view(n, c, X2, 2, Y2, 2, Z2, 2).permute(0, 2, 4, 6, 3, 5, 7, 1).reshape(n, X2, Y2, Z2, 32)
    zero = torch.zeros_like(b[:, :, :, :1])
    lo = torch.cat([zero, b], 3)          # block k-1 at row k
    hi = torch.cat([b, zero], 3)          # block k   at row k
    return torch.cat([lo, hi], -1)


def emulate_conv(x, w_packed, taps, shift, out_dims, stride=1, relu=False, res=None):
    """x (N,X,Y,Z,Cin) float, w_packed (taps,CoutPad,Cin) float -> (N,Xo,Yo,Zo,CoutPad) float."""
    n, X, Y, Z, cin = x.shape
    xo, yo, zo = out_dims
    out = torch.zeros((n, xo, yo, zo, w_packed.shape[1]), dtype=torch.float32, device=x.device)
    P = 8
    xp = F.pad(x, (0, 0, P, P + xo * stride, P, P + yo * stride, P, P + zo * stride))
    for t, (dx, dy, dz) in enumerate(taps):
        sl = xp[:, P + dx: P + dx + xo * stride: stride, P + dy: P + dy + yo * stride: stride,
                P + dz: P + dz + zo * stride: stride]
        out += sl.float() @ w_packed[t].float().t()
    out = out + shift.float()
    if res is not None:
        r = res.float()
        if r.shape[1:4] != out.shape[1:4]:
            r = F.interpolate(r.permute(0, 4, 1, 2, 3), size=(xo, yo, zo), mode="nearest").permute(0, 2, 3, 4, 1)
        out[..., : r.shape[-1]] += r
    if relu:
        out = out.clamp_min(0)
    return out


def nearest_source_index(out_size: int, in_size: int, device=None) -> torch.Tensor:
    """Source index of each output index of a nearest up-sampling from in_size to out_size, as the kernel (row_pos) and
    F.interpolate(mode='nearest', size=...) compute it: min(floor(float32(o) * float32(in / out)), in - 1), all in float32.
    A float64 ratio can pick a different voxel (in 14 -> out 46: output 23 takes voxel 6, not 7)."""
    scale = torch.tensor(float(in_size), dtype=torch.float32) / torch.tensor(float(out_size), dtype=torch.float32)
    idx = torch.floor(torch.arange(out_size, dtype=torch.float32) * scale).to(torch.int64).clamp_max(in_size - 1)
    return idx.to(device)


def reference_conv64(x, w, taps, shift, out_dims, stride=1, act=0, res=None):
    """float64 statement of nrpn_conv3d_fprop on the exact operands the kernel reads (CPU or GPU).

    x (N,X,Y,Z,Cin) 16-bit; w the packed weights, (taps,CoutPad,Cin) or wsplit (taps,2,CoutPad,Cin) whose hi + lo planes are
    summed in float64; shift (CoutPad) fp32; res None or (N,Xr,Yr,Zr,C) 16-bit, nearest-upsampled when its extent differs from
    out_dims and added to the first C channels; act 0 none, 1 ReLU, 2 exact (erf) GELU.
    Returns (ref, mag), float64 (N,Xo,Yo,Zo,CoutPad): ref the result; mag the same sum taken over the absolute value of every
    term (|x|.|w| products, |shift|, |res|, before the activation) -- the scale of the rounding error of a float accumulation."""
    dev = x.device
    x = x.double()
    w = w.double()
    wabs = w.abs()
    if w.dim() == 4:
        w, wabs = w[:, 0] + w[:, 1], wabs[:, 0] + wabs[:, 1]
    n, X, Y, Z, cin = x.shape
    out_dims = tuple(int(v) for v in out_dims)
    P = max(max(abs(int(v)) for v in t) for t in taps)
    hi = [max(0, P + (o - 1) * stride + 1 - i) for o, i in zip(out_dims, (X, Y, Z))]
    xp = F.pad(x, (0, 0, P, hi[2], P, hi[1], P, hi[0]))
    xa = xp.abs()
    ref = torch.zeros((n, *out_dims, w.shape[1]), dtype=torch.float64, device=dev)
    mag = torch.zeros_like(ref)
    xo, yo, zo = out_dims
    for t, (dx, dy, dz) in enumerate(taps):
        ix = slice(P + dx, P + dx + (xo - 1) * stride + 1, stride)
        iy = slice(P + dy, P + dy + (yo - 1) * stride + 1, stride)
        iz = slice(P + dz, P + dz + (zo - 1) * stride + 1, stride)
        ref += xp[:, ix, iy, iz] @ w[t].t()
        mag += xa[:, ix, iy, iz] @ wabs[t].t()
    s = shift.to(dev).double()
    ref += s
    mag += s.abs()
    if res is not None:
        r = res.double()
        if tuple(r.shape[1:4]) != out_dims:
            r = r[:, nearest_source_index(xo, r.shape[1], dev)]
            r = r[:, :, nearest_source_index(yo, r.shape[2], dev)]
            r = r[:, :, :, nearest_source_index(zo, r.shape[3], dev)]
        c = r.shape[-1]
        ref[..., :c] += r
        mag[..., :c] += r.abs()
    if act == 1:
        ref = ref.clamp_min(0)
    elif act == 2:
        ref = 0.5 * ref * (1.0 + torch.erf(ref / math.sqrt(2.0)))
    return ref, mag


def reference_wgrad64(dys, xs, taps, x_dims=None):
    """float64 statement of nrpn_conv3d_wgrad on the exact operands the kernel reads (CPU or GPU):
        dW[tap][co][ci] = sum over levels, samples and voxels v of dY   dY[v][co] * X[v + tap][ci],   X zero outside its grid.

    dys / xs: one (N,X,Y,Z,Cout) / (N,X',Y',Z',Cin) 16-bit tensor per level (the real channels: slice away any row padding).
    x_dims: per level, the extent of X when it differs from dY's (the descriptor's xx / xy / xz); without it X must have dY's extent.
    Returns (ref, mag), float64 (taps, Cout, Cin): mag is the same sum over |dY| |X| -- the scale of the rounding error of a float
    accumulation."""
    cout, cin = dys[0].shape[-1], xs[0].shape[-1]
    P = max(max(abs(int(v)) for v in t) for t in taps)
    ref = torch.zeros((len(taps), cout, cin), dtype=torch.float64, device=dys[0].device)
    mag = torch.zeros_like(ref)
    for i, (dy, x) in enumerate(zip(dys, xs)):
        ext, xext = tuple(dy.shape[1:4]), tuple(x.shape[1:4])
        want = ext if x_dims is None else tuple(x_dims[i])
        assert xext == want and dy.shape[0] == x.shape[0], f"level {i}: X extent {xext}, expected {want}"
        d = dy.double().reshape(-1, cout)
        da = d.abs()
        hi = [max(0, P + e - xe) for e, xe in zip(ext, xext)]
        xp = F.pad(x.double(), (0, 0, P, hi[2], P, hi[1], P, hi[0]))
        xa = xp.abs()
        for t, (dx, dy_, dz) in enumerate(taps):
            sl = (slice(None), slice(P + dx, P + dx + ext[0]), slice(P + dy_, P + dy_ + ext[1]), slice(P + dz, P + dz + ext[2]))
            ref[t] += d.t() @ xp[sl].reshape(-1, cin)
            mag[t] += da.t() @ xa[sl].reshape(-1, cin)
    return ref, mag


def _relative_position_index() -> torch.Tensor:
    """(64 * 64) index into the 343-row relative-position bias table of a 4^3 window, query-major, as the model builds it."""
    from nerf_rpn_b200.model.feature_extractor import ShiftedWindowAttention
    return ShiftedWindowAttention(32, [4, 4, 4], [0, 0, 0], 1).relative_position_index.clone()


def reference_window_attention64(qkv, qkv_bias, table, heads, shift, fmt, flaw=None):
    """float64 statement of nrpn_window_attention on the exact operands the kernel reads (CPU or GPU).

    qkv (N,H,W,D,ld) 16-bit holding [q | k | v] in its first 3C columns (C = 32 heads, head-major); qkv_bias (3C) fp32;
    table (343, heads) fp32; fmt the 16-bit format.  Zero-padded tokens enter the qkv Linear as zeros, so they carry qkv_bias --
    rounded to fmt, as the kernel packs it (real tokens reach it already rounded by the qkv GEMM).  Pad to multiples of 4,
    roll by -shift on every axis whose padded extent exceeds 4, split into 4^3 windows, softmax(q.k / sqrt(32) + relative-
    position bias - 100 between tokens of different shift regions) . v, roll back, crop.
    Returns (ref, scale), float64 (N,H,W,D,C): scale = sum_j p_j |v_j|, the magnitude the rounding of p scales with.
    flaw: a deliberate mistake, for the negative controls of tests/test_norm_attention_reference_cpu.py -- "mask_h_omitted"
    (no region split along H), "mask_unshifted_axes" (regions of the requested shift on every axis), "index_transposed"
    (bias of j - i instead of i - j), "pad_zero" (padding tokens zero instead of the bias), "no_scale" (no 1/sqrt(32))."""
    n, H, W, D, _ = qkv.shape
    C, dev, win = heads * 32, qkv.device, 4
    PH, PW, PD = (-(-e // win) * win for e in (H, W, D))
    sh = [0 if win >= e else shift for e in (PH, PW, PD)]
    bias = qkv_bias.to(dev).to(fmt).double()
    if flaw == "pad_zero":
        bias = torch.zeros_like(bias)
    xp = bias.expand(n, PH, PW, PD, 3 * C).clone()
    xp[:, :H, :W, :D] = qkv[..., :3 * C].double()
    xp = torch.roll(xp, shifts=(-sh[0], -sh[1], -sh[2]), dims=(1, 2, 3))
    nh, nw, nd = PH // win, PW // win, PD // win
    t = xp.view(n, nh, win, nw, win, nd, win, 3 * C).permute(0, 1, 3, 5, 2, 4, 6, 7).reshape(-1, 64, 3, heads, 32)
    q, k, v = t.permute(2, 0, 3, 1, 4)                      # (windows, heads, 64, 32) each
    if flaw != "no_scale":
        q = q * 32 ** -0.5
    attn = q @ k.transpose(-2, -1)
    idx = _relative_position_index()
    if flaw == "index_transposed":
        idx = idx.view(64, 64).t().reshape(-1)
    attn = attn + table.to(dev).double()[idx.to(dev)].view(64, 64, heads).permute(2, 0, 1)
    if sum(sh) > 0:
        mask_sh = [shift] * 3 if flaw == "mask_unshifted_axes" else sh
        labels = []
        for axis, (P, s) in enumerate(zip((PH, PW, PD), mask_sh)):
            lab = torch.zeros(P, dtype=torch.float64, device=dev)
            for r, (lo, hi) in enumerate(((0, -win), (-win, -s), (-s, None))):   # s == 0: (-4, -0) is empty, (-0, None) all
                lab[lo:hi] = r
            if flaw == "mask_h_omitted" and axis == 0:
                lab.zero_()
            labels.append(lab)
        region = labels[0].view(-1, 1, 1) * 9 + labels[1].view(1, -1, 1) * 3 + labels[2].view(1, 1, -1)
        region = region.view(nh, win, nw, win, nd, win).permute(0, 2, 4, 1, 3, 5).reshape(-1, 64)
        mask = (region[:, :, None] != region[:, None, :]).double() * -100.0
        attn = (attn.view(n, -1, heads, 64, 64) + mask[None, :, None]).view(-1, heads, 64, 64)
    p = torch.softmax(attn, dim=-1)

    def unwindow(o):
        o = o.transpose(1, 2).reshape(n, nh, nw, nd, win, win, win, C).permute(0, 1, 4, 2, 5, 3, 6, 7).reshape(n, PH, PW, PD, C)
        return torch.roll(o, shifts=tuple(sh), dims=(1, 2, 3))[:, :H, :W, :D].contiguous()
    return unwindow(p @ v), unwindow(p @ v.abs())


def _normalize64(x, dims, eps, unbiased=False, amplify=False):
    """float64 x normalised over `dims` with the biased variance (the unbiased one only as a negative control).  Returns
    (x_hat, mag): mag = |x_hat| a + mean|x| / sigma, a = E[x^2] / (var + eps) if amplify else 1 -- what an fp32 statistic's
    relative error is multiplied by on its way to the output (divided by |gamma|)."""
    cnt = math.prod(x.shape[d] for d in dims)
    mu = x.mean(dims, keepdim=True)
    d = x - mu
    var = (d * d).sum(dims, keepdim=True) / (cnt - 1 if unbiased else cnt)
    sigma = torch.sqrt(var + eps)
    xh = d / sigma
    a = (x * x).mean(dims, keepdim=True) / (var + eps) if amplify else 1.0
    return xh, xh.abs() * a + x.abs().mean(dims, keepdim=True) / sigma


def reference_layernorm64(x, C, gamma, beta, eps, flaw=None):
    """float64 statement of nrpn_layernorm: LayerNorm over the first C channels of each row of x (..., ld), 16-bit; the
    channels [C, ld) are not read.  Returns (ref, scale), float64 (..., C): scale = |gamma| (|x_hat| + mean|x| / sigma) + |beta|,
    the magnitude the fp32 statistics' and the affine step's rounding scale with.  flaw "unbiased": variance over C - 1."""
    xh, mag = _normalize64(x[..., :C].double(), (-1,), eps, unbiased=flaw == "unbiased")
    g, b = gamma.to(x.device).double(), beta.to(x.device).double()
    return xh * g + b, mag * g.abs() + b.abs()


MERGE_PARITY = ((0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0), (0, 0, 1), (1, 0, 1), (0, 1, 1), (1, 1, 1))


def reference_patch_merge64(x, C, gamma, beta, eps, flaw=None):
    """float64 statement of nrpn_patch_merge_ln: x (N,H,W,D,ld) 16-bit, first C channels read; output token (i,j,k) is the
    LayerNorm(8C) of the input tokens (2i+a, 2j+b, 2k+c) concatenated in parity order 000,100,010,110,001,101,011,111 (over H,W,D),
    zero past an odd extent.  Returns (ref, scale) as reference_layernorm64, (N, ceil(H/2), ceil(W/2), ceil(D/2), 8C).
    flaw: "swap_100_010" (those two parts exchanged), "edge_replicate" (the last plane repeated past an odd extent)."""
    xs = x[..., :C].double()
    for axis in (1, 2, 3):
        if xs.shape[axis] % 2:
            edge = xs.narrow(axis, xs.shape[axis] - 1, 1)
            xs = torch.cat([xs, edge if flaw == "edge_replicate" else torch.zeros_like(edge)], axis)
    order = list(MERGE_PARITY)
    if flaw == "swap_100_010":
        order[1], order[2] = order[2], order[1]
    merged = torch.cat([xs[:, a::2, b::2, c::2] for a, b, c in order], -1)
    return reference_layernorm64(merged, 8 * C, gamma, beta, eps)


def reference_groupnorm64(levels, gamma, beta, eps, relu, flaw=None):
    """float64 statement of nrpn_groupnorm_relu: levels a list of (N, ..., 256) 16-bit tensors; 32 groups of 8 consecutive
    channels; mean and biased variance per (sample, level, group) over the group's channels and every voxel; then
    x_hat gamma + beta, and ReLU if relu.  Returns (refs, scales), lists of float64 (N, ..., 256):
    scale = |gamma| (|x_hat| E[x^2] / (var + eps) + mean|x| / sigma) + |beta| (before the ReLU) -- the kernel forms the variance
    as E[x^2] - mean^2, so a relative error of E[x^2] reaches the output multiplied by E[x^2] / var.
    flaw: "unbiased" (variance over count - 1), "group_mod32" (channel c in group c % 32), "pooled" (statistics over all samples)."""
    refs, scales = [], []
    for x in levels:
        n, shape = x.shape[0], x.shape
        xs = x.double().reshape(n, -1, 256)
        if flaw == "group_mod32":
            g = xs.view(n, -1, 8, 32)                                # group = c % 32: the last index
            dims = (1, 2)
        else:
            g = xs.view(n, -1, 32, 8)                                # group = c // 8
            dims = (1, 3)
        if flaw == "pooled":
            dims = (0,) + dims
        xh, mag = _normalize64(g, dims, eps, unbiased=flaw == "unbiased", amplify=True)
        xh, mag = xh.reshape(shape), mag.reshape(shape)
        ga, be = gamma.to(x.device).double(), beta.to(x.device).double()
        y = xh * ga + be
        refs.append(y.clamp_min(0) if relu else y)
        scales.append(mag * ga.abs() + be.abs())
    return refs, scales


def reference_patch_embed(grid):
    """nrpn_patch_embed_pack: fp32 (N,4,X,Y,Z) -> float64 (N, X/4, Y/4, Z/4, 256), row (i,j,k) channel ((c*4+px)*4+py)*4+pz =
    grid[c][4i+px][4j+py][4k+pz] (remainders of X, Y, Z past a multiple of 4 unused) -- the patch embedding Conv3d(4, C, 4,
    stride 4) as a 256 -> C GEMM with the weight flattened in (c, px, py, pz) order.  Exact: compare it bit for bit after
    rounding to the 16-bit format."""
    n, c, X, Y, Z = grid.shape
    H, W, D = X // 4, Y // 4, Z // 4
    g = grid[:, :, :4 * H, :4 * W, :4 * D].double().reshape(n, c, H, 4, W, 4, D, 4)
    return g.permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(n, H, W, D, 256)


def emulate_pack_stem_s1(grid: torch.Tensor) -> torch.Tensor:
    """(N,4,X,Y,Z) -> (N,X,Y+1,Z,64) with the layout of csrc/pointwise.cu:pack_stem_s1_kernel."""
    n, c, X, Y, Z = grid.shape
    g = F.pad(grid, (3, 3, 1, 1))                       # z by 3, y by 1 on both sides
    out = torch.zeros((n, X, Y + 1, Z, 64), dtype=grid.dtype, device=grid.device)
    for yy in range(2):
        for zz in range(7):
            # row yp holds input y = yp - 1 + yy  -> padded index yp + yy ; z neighbour z + zz - 3 -> padded z + zz
            sl = g[:, :, :, yy: yy + Y + 1, zz: zz + Z]                 # (n, c, X, Y+1, Z)
            ch = (yy * 7 + zz) * 4
            out[..., ch:ch + 4] = sl.permute(0, 2, 3, 4, 1)
    return out


# ------------------------------------------------------------------------------------------------ training-step bandwidth kernels
# float64 statements of what csrc/train.cu (and the poolings / stride-1 stem packing of csrc/pointwise.cu) compute, on the exact 16-bit or
# fp32 operands the kernels read.  Each returns the result and, where the kernel rounds in float arithmetic, the magnitude that rounding
# scales with.  `flaw` selects a deliberate mistake, for the negative controls of tests/test_bandwidth_reference_cpu.py.

def reference_bn_stats64(y, eps, running_mean=None, running_var=None, momentum=0.1, chunk=1 << 18, flaw=None):
    """nrpn_bn_stats: y (rows, C) 16-bit.  Batch mean and biased variance per channel (two passes, float64, `chunk` rows at a time),
    rstd = 1 / sqrt(var + eps), and the running-stat update of nn.BatchNorm3d in train mode: r = (1 - momentum) r + momentum s, with
    the unbiased variance var * rows / (rows - 1).  Returns a dict of float64 (C) tensors: mean, var, rstd, e_abs = E|y|, e_sq = E[y^2],
    and running_mean / running_var (updated copies) when given.  flaw "biased_running_var": the running variance takes the biased one."""
    rows, c = y.shape
    s1 = torch.zeros(c, dtype=torch.float64, device=y.device)
    sa, s2 = torch.zeros_like(s1), torch.zeros_like(s1)
    for r0 in range(0, rows, chunk):
        v = y[r0:r0 + chunk].double()
        s1 += v.sum(0)
        sa += v.abs().sum(0)
        s2 += (v * v).sum(0)
    mean = s1 / rows
    sd = torch.zeros_like(s1)
    for r0 in range(0, rows, chunk):
        d = y[r0:r0 + chunk].double() - mean
        sd += (d * d).sum(0)
    var = sd / rows
    out = dict(mean=mean, var=var, rstd=1.0 / torch.sqrt(var + eps), e_abs=sa / rows, e_sq=s2 / rows)
    if running_mean is not None:
        unbiased = var if flaw == "biased_running_var" or rows == 1 else var * rows / (rows - 1)
        out["running_mean"] = (1.0 - momentum) * running_mean.double() + momentum * mean
        out["running_var"] = (1.0 - momentum) * running_var.double() + momentum * unbiased
    return out


def reference_bn_apply64(y, res, mean, rstd, gamma, beta, relu):
    """nrpn_bn_apply: out = act(gamma (y - mean) rstd + beta (+ res)) for y, res (rows, C) 16-bit and the fp32 per-channel mean, rstd
    (the statistics the kernel reads), gamma, beta.  Returns (ref, scale): scale = |gamma x_hat| + |beta| + |res|, what the fp32
    multiply-adds round relative to."""
    dev = y.device
    xh = (y.double() - mean.to(dev).double()) * rstd.to(dev).double()
    g, b = gamma.to(dev).double(), beta.to(dev).double()
    ref = xh * g + b
    scale = (xh * g).abs() + b.abs()
    if res is not None:
        ref = ref + res.double()
        scale = scale + res.double().abs()
    return (ref.clamp_min(0) if relu else ref), scale


def reference_bn_backward64(dout, act, y, mean, rstd, gamma, relu, sums=None, rows=None, flaw=None):
    """nrpn_bn_backward on dout, act (the forward's 16-bit output, read only for the ReLU mask), y (rows, C) 16-bit and the fp32
    statistics mean, rstd the kernel reads: g = dout * (act > 0 if relu), x_hat = (y - mean) rstd,
      dgamma = sum g x_hat,  dbeta = sum g,  dy = gamma rstd (g - dbeta / M - x_hat dgamma / M),  dres = g.
    dy is stated on `sums` = (dgamma, dbeta) as the kernel read them (its own fp32 output) when given, else on the float64 sums;
    `rows` = M, the rows of the whole batch when these are a slice of it (default: y's rows).
    Returns a dict of float64: dgamma, dbeta (C) and their magnitudes mag_dgamma = sum |g x_hat|, mag_dbeta = sum |g|; dy, dres
    (rows, C) and mag_dy = |gamma rstd| (|g| + |dbeta| / M + |x_hat dgamma| / M).
    flaw "relu_mask_dropped": g = dout everywhere; "dres_unmasked": dres = dout."""
    dev = y.device
    rows = y.shape[0] if rows is None else rows
    d = dout.double()
    g = d * (act > 0).double() if relu and flaw != "relu_mask_dropped" else d
    xh = (y.double() - mean.to(dev).double()) * rstd.to(dev).double()
    out = dict(dgamma=(g * xh).sum(0), dbeta=g.sum(0), mag_dgamma=(g * xh).abs().sum(0), mag_dbeta=g.abs().sum(0))
    sg, sb = (out["dgamma"], out["dbeta"]) if sums is None else (s.to(dev).double() for s in sums)
    k = gamma.to(dev).double() * rstd.to(dev).double()
    out["dy"] = k * (g - sb / rows - xh * sg / rows)
    out["mag_dy"] = k.abs() * (g.abs() + sb.abs() / rows + (xh * sg).abs() / rows)
    out["dres"] = d if flaw == "dres_unmasked" else g
    return out


MAXPOOL3_TAPS = [(dx, dy, dz) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1)]     # scan order: x outer, z inner


def reference_maxpool3_argmax(x, flaw=None):
    """nrpn_maxpool3d_k3s2_argmax / nrpn_maxpool3d_k3s2: F.max_pool3d(kernel 3, stride 2, padding 1) of x (N,X,Y,Z,C) 16-bit, and the
    window position (dx+1)*9 + (dy+1)*3 + (dz+1) of the FIRST maximum in scan order (x outer, z inner; padded taps never win), the
    element torch's max_pool3d_with_indices records.  Exact: returns (out in x's dtype, code uint8).  flaw "last_max": the last."""
    n, X, Y, Z, C = x.shape
    Xo, Yo, Zo = ((e - 1) // 2 + 1 for e in (X, Y, Z))
    xp = F.pad(x.float(), (0, 0, 1, 2 * Zo - Z, 1, 2 * Yo - Y, 1, 2 * Xo - X), value=-math.inf)
    best = torch.full((n, Xo, Yo, Zo, C), -math.inf, device=x.device)
    code = torch.full((n, Xo, Yo, Zo, C), 13, dtype=torch.uint8, device=x.device)
    for t, (dx, dy, dz) in enumerate(MAXPOOL3_TAPS):
        v = xp[:, 1 + dx: 1 + dx + 2 * Xo: 2, 1 + dy: 1 + dy + 2 * Yo: 2, 1 + dz: 1 + dz + 2 * Zo: 2]
        take = (v >= best) & (v > -math.inf) if flaw == "last_max" else v > best
        best = torch.where(take, v, best)
        code[take] = t
    return best.to(x.dtype), code


def reference_maxpool3_backward64(dy, code, in_dims):
    """nrpn_maxpool3d_k3s2_backward: input voxel 2 o + (d - 1) of each output o receives dy[o] when code[o] names its window position d.
    dy (N,Xo,Yo,Zo,C) 16-bit, code uint8 as the forward wrote it.  Returns (ref, mag) float64 (N,X,Y,Z,C): mag = the sum of |dy|."""
    n, Xo, Yo, Zo, C = dy.shape
    X, Y, Z = in_dims
    ref = torch.zeros((n, 2 * Xo + 2, 2 * Yo + 2, 2 * Zo + 2, C), dtype=torch.float64, device=dy.device)
    mag = torch.zeros_like(ref)
    d = dy.double()
    for t, (dx, dy_, dz) in enumerate(MAXPOOL3_TAPS):
        v = torch.where(code == t, d, torch.zeros_like(d))
        sl = (slice(None), slice(1 + dx, 1 + dx + 2 * Xo, 2), slice(1 + dy_, 1 + dy_ + 2 * Yo, 2), slice(1 + dz, 1 + dz + 2 * Zo, 2))
        ref[sl] += v
        mag[sl] += v.abs()
    crop = (slice(None), slice(1, 1 + X), slice(1, 1 + Y), slice(1, 1 + Z))
    return ref[crop], mag[crop]


def reference_maxpool2_ceil(x):
    """nrpn_maxpool3d_k2s2_ceil: nn.MaxPool3d(2, 2, ceil_mode=True) of x (N,X,Y,Z,C) 16-bit, the last window clipped at an odd
    extent.  Exact: returns x's dtype, (N, ceil(X/2), ceil(Y/2), ceil(Z/2), C)."""
    n, X, Y, Z, C = x.shape
    xp = F.pad(x.float(), (0, 0, 0, Z % 2, 0, Y % 2, 0, X % 2), value=-math.inf)
    out = None
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                v = xp[:, dx::2, dy::2, dz::2]
                out = v if out is None else torch.maximum(out, v)
    return out.to(x.dtype)


def reference_upsample_backward64(dfine, dcoarse, flaw=None):
    """nrpn_upsample_nearest_backward: dcoarse + the backward of the nearest up-sampling coarse -> fine (F.interpolate(mode='nearest',
    size=fine)): each fine voxel's gradient goes to the coarse voxel nearest_source_index picks on every axis.  dfine (N,Xf,Yf,Zf,C),
    dcoarse (N,Xc,Yc,Zc,C) 16-bit.  Returns (ref, mag, terms): mag = |dcoarse| + the sum of |dfine|, terms the most fine voxels one
    coarse voxel collects.  flaw "float64_index": floor(o * in / out) in float64."""
    dev = dfine.device
    ref, mag = dfine.double(), dfine.double().abs()
    terms = 1
    for axis in (1, 2, 3):
        fo, ci = dfine.shape[axis], dcoarse.shape[axis]
        if flaw == "float64_index":
            idx = torch.tensor([min(int(math.floor(o * ci / fo)), ci - 1) for o in range(fo)], device=dev)
        else:
            idx = nearest_source_index(fo, ci, dev)
        terms *= int(torch.bincount(idx, minlength=ci).max())
        shape = list(ref.shape)
        shape[axis] = ci
        ref = torch.zeros(shape, dtype=torch.float64, device=dev).index_add_(axis, idx, ref)
        mag = torch.zeros(shape, dtype=torch.float64, device=dev).index_add_(axis, idx, mag)
    return ref + dcoarse.double(), mag + dcoarse.double().abs(), terms


def rpn_anchors_f32(flat, level_dims, strides, cells, A):
    """The anchors nrpn_rpn_loss derives from flat anchor indices (levels in order, then voxel x-major, then anchor a), in float32 as
    the kernel forms them: (x * stride + cell[a][k]) per coordinate.  flat int64 (S,); cells per level (A, 6).  Returns (level, vox,
    a, anchors (S, 6) float32)."""
    dev = flat.device
    begin = [0]
    for d in level_dims:
        begin.append(begin[-1] + d[0] * d[1] * d[2] * A)
    lvl = torch.zeros_like(flat)
    for l in range(1, len(level_dims)):
        lvl += (flat >= begin[l]).long()
    r = flat - torch.tensor(begin[:-1], device=dev)[lvl]
    a, vox = r % A, r // A
    gx, gy, gz = (torch.tensor([d[k] for d in level_dims], device=dev)[lvl] for k in range(3))
    z, y, x = vox % gz, (vox // gz) % gy, vox // (gz * gy)
    st = torch.tensor(strides, device=dev)[lvl]
    cell = torch.stack([torch.as_tensor(c, dtype=torch.float32) for c in cells]).to(dev)[lvl, a]
    base = torch.stack([x * st[:, 0], y * st[:, 1], z * st[:, 2]], 1).float()
    return lvl, vox, a, torch.cat([base, base], 1) + cell


def encode_targets64(anchors, gt, rotated):
    """The RPN box encoders of nrpn_rpn_loss in float64 on the float32 anchors (S,6) and gt (S,6|7): AABB_coder.encode_boxes_3d, or
    midpoint_offset bbox2delta_sp whose cos / sin, polygon and vertex selection (|coordinate - extreme| > 0.1) are taken in float32
    exactly as oracle/loss_oracle.py does (a float64 polygon would flip vertices near the threshold), then float64.  Returns (t, mag):
    mag = (sum of the |coordinates| and sizes read) / the smallest size divided by + |t| + 1, what the kernel's fp32 rounding of the
    coordinates reaches each delta with."""
    an, g = anchors.double(), gt.double()
    asz = an[:, 3:] - an[:, :3]
    if not rotated:
        gsz = g[:, 3:] - g[:, :3]
        t = torch.cat([((g[:, :3] + 0.5 * gsz) - (an[:, :3] + 0.5 * asz)) / asz, torch.log(gsz / asz)], 1)
        size = torch.cat([asz, gsz], 1).min(1).values
        coords = an.abs().sum(1) + g.abs().sum(1)
    else:
        gf = gt.float()
        x, y, w, h, th = gf[:, 0], gf[:, 1], gf[:, 3], gf[:, 4], gf[:, 6]
        co, si = torch.cos(th), torch.sin(th)
        v1x, v1y, v2x, v2y = w / 2 * co, -(w / 2) * si, -(h / 2) * si, -(h / 2) * co
        px = torch.stack([x + v1x + v2x, x + v1x - v2x, x - v1x - v2x, x - v1x + v2x], 1)
        py = torch.stack([y + v1y + v2y, y + v1y - v2y, y - v1y - v2y, y - v1y + v2y], 1)
        far = torch.tensor(-1000.0, device=gt.device)
        ga = torch.where((py - py.min(1, keepdim=True).values).abs() > 0.1, far, px).max(1).values.double()
        gb = torch.where((px - px.max(1, keepdim=True).values).abs() > 0.1, far, py).max(1).values.double()
        cd, sd = co.double(), si.double()
        xb = (g[:, 3] / 2 * cd).abs() + (g[:, 4] / 2 * sd).abs()
        yb = (g[:, 3] / 2 * sd).abs() + (g[:, 4] / 2 * cd).abs()
        gw, gh = 2 * xb, 2 * yb
        ctr = (an[:, :3] + an[:, 3:]) * 0.5
        t = torch.stack([(g[:, 0] - ctr[:, 0]) / asz[:, 0], (g[:, 1] - ctr[:, 1]) / asz[:, 1], (g[:, 2] - ctr[:, 2]) / asz[:, 2],
                         torch.log(gw / asz[:, 0]), torch.log(gh / asz[:, 1]), torch.log(g[:, 5] / asz[:, 2]),
                         (ga - g[:, 0]) / gw, (gb - g[:, 1]) / gh], 1)
        size = torch.stack([asz.min(1).values, gw, gh, g[:, 5]], 1).min(1).values
        coords = an.abs().sum(1) + g[:, :6].abs().sum(1) + xb + yb
    return t, (coords / size).unsqueeze(1) + t.abs() + 1.0


def reference_rpn_loss64(pred_rows_pos, logits, n_pos, targets, norm, w_obj, w_reg, grad_scale, flaw=None):
    """nrpn_rpn_loss for one call: logits (S,) fp32 of the sampled anchors, the first n_pos positive (label 1), the rest negative;
    pred_rows_pos (n_pos, code) fp32 the predicted deltas of the positives; targets (n_pos, code) float64 (encode_targets64).
      L_obj = sum BCE-with-logits / norm,  L_reg = sum smooth-L1(beta 1/9) / norm  (norm = sampled anchors of the whole batch)
      dlogit = (sigmoid(x) - y) / norm * w_obj * grad_scale,  ddelta = smooth-L1'(p - t) / norm * w_reg * grad_scale.
    Returns a dict of float64: l_obj, l_reg, dlogit (S,), ddelta (n_pos, code), and the magnitudes for the bounds: mag_obj (S,) = |x| + 1
    per BCE term, d (n_pos, code) = p - t.  flaw "beta_1": smooth-L1 with beta 1; "bce_over_positives": BCE normalised by n_pos."""
    x = logits.double()
    lab = torch.zeros_like(x)
    lab[:n_pos] = 1.0
    beta = 1.0 if flaw == "beta_1" else 1.0 / 9.0
    bce = x.clamp_min(0) - x * lab + torch.log1p(torch.exp(-x.abs()))
    obj_norm = float(max(n_pos, 1)) if flaw == "bce_over_positives" else norm
    d = pred_rows_pos.double() - targets
    ad = d.abs()
    sl1 = torch.where(ad < beta, 0.5 * d * d / beta, ad - 0.5 * beta)
    gr = torch.where(ad < beta, d / beta, torch.sign(d))
    return dict(l_obj=float(bce.sum()) / obj_norm, l_reg=float(sl1.sum()) / norm,
                dlogit=(torch.sigmoid(x) - lab) / obj_norm * w_obj * grad_scale, ddelta=gr / norm * w_reg * grad_scale,
                mag_obj=x.abs() + 1.0, d=d)


def reference_grad_norm64(g, inv_scale):
    """nrpn_grad_norm: sqrt(sum g^2) * inv_scale over the fp32 gradient g, float64."""
    s = 0.0
    for i in range(0, g.numel(), 1 << 24):
        v = g[i:i + (1 << 24)].double()
        s += float((v * v).sum())
    return math.sqrt(s) * inv_scale


def reference_adamw64(p, g, m, v, norm, max_norm, inv_scale, lr, beta1, beta2, eps, wd, step, flaw=None):
    """nrpn_adamw_step in float64 on its fp32 operands, norm the fp32 gradient norm it reads: torch.nn.utils.clip_grad_norm_ (coefficient
    min(max_norm / (norm + 1e-6), 1), none when max_norm <= 0) on the gradient g * inv_scale, then one torch.optim.AdamW step:
      p <- p (1 - lr wd),  m <- b1 m + (1 - b1) g,  v <- b2 v + (1 - b2) g^2,  p <- p - lr / (1 - b1^t) * m / (sqrt(v / (1 - b2^t)) + eps).
    Returns (p, m, v, u) float64: u = lr / (1 - b1^t) * |m| / (sqrt(v / (1 - b2^t)) + eps), the size of the update.
    flaw "no_bias_correction", "l2_decay" (wd p added to the gradient instead of decoupled), "unclamped_clip" (no min(., 1))."""
    coef = inv_scale
    if max_norm > 0:
        c = max_norm / (float(norm) + 1e-6)
        coef *= c if flaw == "unclamped_clip" else min(c, 1.0)
    p, g, m, v = (t.double() for t in (p, g, m, v))
    gi = g * coef
    if flaw == "l2_decay":
        gi = gi + wd * p
    else:
        p = p * (1.0 - lr * wd)
    m = beta1 * m + (1.0 - beta1) * gi
    v = beta2 * v + (1.0 - beta2) * gi * gi
    bc1, bc2 = (1.0, 1.0) if flaw == "no_bias_correction" else (1.0 - beta1 ** step, 1.0 - beta2 ** step)
    u = lr / bc1 * m / (torch.sqrt(v / bc2) + eps)
    return p - u, m, v, u.abs()

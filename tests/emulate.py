"""Pure-torch statement of what nrpn_conv3d_fprop / nrpn_conv3d_wgrad / nrpn_pack_stem_input and the Swin-3D / GroupNorm kernels compute (TEST
helper, CPU or GPU).  Used to check the host-side packing logic without a GPU and as the fp32 / float64 references for the CUDA
kernels."""
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

"""Pure-torch statement of what nrpn_conv3d_fprop / nrpn_pack_stem_input compute (TEST helper, CPU or GPU).
Used to check the host-side packing logic without a GPU and as the fp32 / float64 references for the CUDA kernels."""
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

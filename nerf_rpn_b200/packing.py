"""Weight pre-packing for the wgmma implicit-GEMM convolution (host-side, runs once per checkpoint).

Reference layouts: nn.Conv3d.weight is (Cout, Cin, kx, ky, kz) fp32 over an NCDHW (N,C,W,L,H) input
(feature_extractor.py:36-43,163,178,184; anchor.py:190-198).  The kernel wants one K-major (Cout x Cin) bf16
matrix per filter tap, (taps, CoutPad, Cin), with eval-mode BatchNorm folded in: scale multiplied into the
weights, shift kept as an fp32 per-channel epilogue add.
"""
from typing import List, Optional, Tuple

import torch


def fold_bn(bn: torch.nn.modules.batchnorm._BatchNorm) -> Tuple[torch.Tensor, torch.Tensor]:
    """eval-mode BatchNorm3d (feature_extractor.py:38,41,43) as y = x * scale + shift."""
    var, mean = bn.running_var.detach().cpu().double(), bn.running_mean.detach().cpu().double()     # host-side, once per checkpoint
    inv = torch.rsqrt(var + bn.eps)
    scale = bn.weight.detach().cpu().double() * inv
    shift = bn.bias.detach().cpu().double() - mean * scale
    return scale.float(), shift.float()


def _round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


def conv_block_n(cout: int) -> int:
    return 64 if cout <= 64 else (128 if cout <= 128 else 256)


def split_hi_lo(w32: torch.Tensor, dtype) -> torch.Tensor:
    """fp32 (..., Cout, Cin) -> 16-bit (..., 2, Cout, Cin): w ~= hi + lo with hi = round16(w), lo = round16(w - hi).  The two planes
    are multiplied with the same activations into one fp32 accumulator (nrpn_conv_desc.wsplit), so the weights keep ~22 bits."""
    hi = w32.to(dtype)
    lo = (w32 - hi.float()).to(dtype)
    return torch.stack([hi, lo], dim=-3).contiguous()


def pack_conv_weight(w: torch.Tensor, scale: Optional[torch.Tensor] = None, cout_pad_to: Optional[int] = None, dtype=torch.bfloat16,
                     split: bool = False):
    """(Cout, Cin, k, k, k) -> (taps, CoutPad, CinPad) bf16 and the tap offset table for 'same' padding (k odd);
    split=True: (taps, 2, CoutPad, CinPad) hi / lo planes (see split_hi_lo)."""
    cout, cin, kx, ky, kz = w.shape
    w = w.detach().float()
    if scale is not None:
        w = w * scale.view(-1, 1, 1, 1, 1).to(w)
    cout8 = _round_up(cout, 8)
    bn = conv_block_n(cout8)
    cpad = _round_up(cout8, bn) if cout_pad_to is None else cout_pad_to
    cin_pad = _round_up(cin, 64)
    taps: List[Tuple[int, int, int]] = []
    mats = []
    for a in range(kx):
        for b in range(ky):
            for c in range(kz):
                taps.append((a - kx // 2, b - ky // 2, c - kz // 2))
                mats.append(w[:, :, a, b, c])
    m = torch.stack(mats, 0)                                   # (taps, Cout, Cin)
    out = torch.zeros((len(taps), cpad, cin_pad), dtype=torch.float32, device=w.device)
    out[:, :cout, :cin] = m
    if split:
        return split_hi_lo(out, dtype), taps
    return out.to(dtype).contiguous(), taps


def pad_shift(shift: torch.Tensor, cpad: int) -> torch.Tensor:
    out = torch.zeros(cpad, dtype=torch.float32, device=shift.device)
    out[: shift.numel()] = shift.detach().float()
    return out


def pack_stem_weight(w: torch.Tensor, scale: Optional[torch.Tensor] = None, dtype=torch.bfloat16):
    """Stem Conv3d(4, 64, kernel 7, stride 2, padding 3) (feature_extractor.py:163) re-expressed on the packed
    space-to-depth input of csrc/pointwise.cu: 4 x 4 x 2 taps, K = 64 per tap.

    Packed row (i,j,k) = [s2d block (i,j,k-1) | s2d block (i,j,k)], block channel = ((rx*2+ry)*2+rz)*4 + c.
    Output voxel o reads input 2*o + kk - 3 (kk = 0..6) = 2*(o + q) + r, q in {-2,-1,0,1}; along z the two blocks of a
    packed row are q = dz-1 and q = dz for tap offset dz in {-1, +1}.
    """
    cout, cin, k, _, _ = w.shape
    assert (cin, k) == (4, 7), "stem packing is specific to the reference's 7^3 stride-2 stem on 4 channels"
    w = w.detach().float()
    if scale is not None:
        w = w * scale.view(-1, 1, 1, 1, 1).to(w)
    taps, mats = [], []
    for qx in (-2, -1, 0, 1):
        for qy in (-2, -1, 0, 1):
            for dz in (-1, 1):
                m = torch.zeros((cout, 64), dtype=torch.float32, device=w.device)
                for half in (0, 1):
                    qz = dz - 1 + half
                    for rx in (0, 1):
                        for ry in (0, 1):
                            for rz in (0, 1):
                                kx, ky, kz = 2 * qx + rx + 3, 2 * qy + ry + 3, 2 * qz + rz + 3
                                if 0 <= kx < 7 and 0 <= ky < 7 and 0 <= kz < 7:
                                    ch = half * 32 + ((rx * 2 + ry) * 2 + rz) * 4
                                    m[:, ch:ch + 4] = w[:, :, kx, ky, kz]
                taps.append((qx, qy, dz))
                mats.append(m)
    out = torch.stack(mats, 0)                                  # (32, 64, 64)
    return out.to(dtype).contiguous(), taps


def pack_stem_s1_weight(w: torch.Tensor, scale: Optional[torch.Tensor] = None, dtype=torch.bfloat16):
    """Stride-1 stem Conv3d(4, 64, kernel 7, padding 3) (VGG_FPN on grids < 160, feature_extractor.py:341) on the packed input
    of csrc/pointwise.cu:pack_stem_s1_kernel: 7 (dx) x 4 (y pairs) taps, K = 64 per tap.

    Packed row (x, yp, z) = rows y = yp-1 and yp, each with its 7 z-neighbours: channel = (yy*7 + zz)*4 + c.
    Output (x,y,z) reads input rows y-3..y+3 = pairs (y+dyp, y+dyp+1) for dyp in {-3,-1,1,3}; pair (a, a+1) lives in packed row
    yp = a+1, so the tap offset in packed coordinates is dyp + 1 (the packed Y extent is Y+1)."""
    cout, cin, k, _, _ = w.shape
    assert (cin, k) == (4, 7)
    w = w.detach().float()
    if scale is not None:
        w = w * scale.view(-1, 1, 1, 1, 1).to(w)
    taps, mats = [], []
    for dx in range(-3, 4):
        for dyp in (-3, -1, 1, 3):
            m = torch.zeros((cout, 64), dtype=torch.float32, device=w.device)
            for yy in (0, 1):
                ky = dyp + yy + 3
                if not 0 <= ky < 7:
                    continue
                for zz in range(7):
                    ch = (yy * 7 + zz) * 4
                    m[:, ch:ch + 4] = w[:, :, dx + 3, ky, zz]
            taps.append((dx, dyp + 1, 0))
            mats.append(m)
    return torch.stack(mats, 0).to(dtype).contiguous(), taps


def pack_conv_weight_dgrad(w: torch.Tensor, dtype=torch.bfloat16):
    """Data-gradient weights of a stride-1 'same' Conv3d: dL/dx = conv(dL/dy, W') with W'[ci, co, a, b, c] = W[co, ci, k-1-a, k-1-b, k-1-c]
    (taps mirrored, matrices transposed), so the backward-data pass of every stride-1 layer runs on the SAME wgmma implicit-GEMM
    kernel as the forward pass (row a18: first building block of the training path; weight gradients need a voxel-major GEMM and
    are not built).  Returns (packed (taps, CinPad, CoutPad... as the kernel's (taps, N, K)), taps)."""
    wt = w.detach().float().permute(1, 0, 2, 3, 4).flip(2, 3, 4).contiguous()
    return pack_conv_weight(wt, None, dtype=dtype)

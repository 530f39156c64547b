"""TEST INFRASTRUCTURE ONLY — float64 references for single launches of the UNet / VAE / CLIP HBM-bound kernels.

Every function here is plain torch on the host (no `dreamllm_b200` import).  Where a kernel rounds to bf16 in the middle of its
formula, the reference rounds at the same point (`bf16r`); the kernel comment that names each rounding point is quoted next to the
function.  tests/test_tower_kernels_cpu.py checks these references against independent torch formulations and autograd;
tests/test_tower_kernels_gpu.py compares the kernels with them.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

BF = torch.bfloat16
F64 = torch.float64


def bf16r(x: torch.Tensor) -> torch.Tensor:
    """Round to bf16 and back to float64 (the kernels' `r16`)."""
    return x.to(torch.float32).to(BF).to(F64)


def bf16_st(x: torch.Tensor) -> torch.Tensor:
    """bf16 rounding in the forward, identity in the backward (a kernel that rounds an intermediate but differentiates the
    unrounded formula)."""
    return x + (bf16r(x) - x).detach()


def _ordered(b: torch.Tensor) -> torch.Tensor:
    i = b.contiguous().view(torch.int16).to(torch.int32)
    return torch.where(i < 0, -(i + 32768), i)


def ulp_diff(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Distance in bf16 units in the last place between two bf16 tensors (+0 and -0 are the same point)."""
    assert a.dtype == BF and b.dtype == BF and a.shape == b.shape
    return (_ordered(a) - _ordered(b)).abs()


# ------------------------------------------------------------------------------------------------ GroupNorm (+SiLU)
def groupnorm_stats(x_nhwc: torch.Tensor, G: int, eps: float):
    """float64 per-(n, g) mean and rstd of x [N, ..., C] (biased variance, as torch.nn.GroupNorm)."""
    N, C = x_nhwc.shape[0], x_nhwc.shape[-1]
    xg = x_nhwc.to(F64).reshape(N, -1, G, C // G)
    mean = xg.mean(dim=(1, 3))
    var = ((xg - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    return mean, (var + eps).rsqrt()


def groupnorm_pre(x_nhwc, w, b, G, eps):
    """float64 (x - mean) * rstd * w + b, before the kernel's bf16 rounding (gn_apply_kernel: `r16(... * wf + bf_)`)."""
    N, C = x_nhwc.shape[0], x_nhwc.shape[-1]
    mean, rstd = groupnorm_stats(x_nhwc, G, eps)
    xg = x_nhwc.to(F64).reshape(N, -1, G, C // G)
    xh = ((xg - mean[:, None, :, None]) * rstd[:, None, :, None]).reshape(x_nhwc.shape)
    return xh * w.to(F64) + b.to(F64)


def groupnorm_silu_ref(x_nhwc, w, b, G, eps, silu):
    """GroupNorm(+SiLU) rounded where gn_apply_kernel rounds: y = silu?(bf16(gn(x) * w + b)); returns float64 (the kernel then rounds
    once more to its bf16 output)."""
    t = bf16r(groupnorm_pre(x_nhwc, w, b, G, eps))
    return F.silu(t) if silu else t


def _from_ordered(o: torch.Tensor) -> torch.Tensor:
    return torch.where(o < 0, -o - 32768, o).to(torch.int16).view(BF)


def neighbour_rounding(pre: torch.Tensor, rel: float = 2.0 ** -16, atol=0.0) -> torch.Tensor:
    """The other bf16 neighbour of `pre` where `pre` lies within `rel * |pre| + atol` of a bf16 rounding midpoint, else bf16r(pre).

    An fp32 kernel that rounds `pre` to bf16 may land on either neighbour there; the float64 reference cannot say which."""
    near = pre.to(torch.float32).to(BF)
    o = _ordered(near)
    up = near.to(F64) <= pre
    other = _from_ordered(torch.where(up, o + 1, o - 1)).to(F64)
    mid = 0.5 * (near.to(F64) + other)
    close = (pre - mid).abs() <= rel * pre.abs() + atol
    return torch.where(close, other, near.to(F64))


def groupnorm_silu_autograd_dx(x_nhwc, w, b, G, eps, silu, dy, dres=None):
    """float64 autograd of silu?(bf16(group_norm(x) * w + b)) w.r.t. x, the bf16 rounding straight-through (what
    groupnorm_bwd_nhwc differentiates: g = dy * silu'(y) * w with y the rounded value)."""
    x = x_nhwc.to(F64).detach().requires_grad_(True)
    N, C = x.shape[0], x.shape[-1]
    xc = x.reshape(N, -1, C).transpose(1, 2)                      # [N, C, HW]
    y = F.group_norm(xc, G, w.to(F64), b.to(F64), eps).transpose(1, 2).reshape(x.shape)
    y = bf16_st(y)
    if silu:
        y = F.silu(y)
    (y * dy.to(F64)).sum().backward()
    dx = x.grad
    return dx + dres.to(F64) if dres is not None else dx


# ------------------------------------------------------------------------------------------------ LayerNorm
def layernorm_ref(x2d, w, b, eps):
    return F.layer_norm(x2d.to(F64), (x2d.shape[-1],), w.to(F64), b.to(F64), eps)


def layernorm_autograd_dx(x2d, w, b, eps, dy, dres=None):
    x = x2d.to(F64).detach().requires_grad_(True)
    (layernorm_ref(x, w, b, eps) * dy.to(F64)).sum().backward()
    return x.grad + dres.to(F64) if dres is not None else x.grad


# ------------------------------------------------------------------------------------------------ GEGLU
def geglu_ref(in2d):
    """out = h * bf16(gelu(gate)) — geglu_kernel rounds gelu(gate) to bf16 before the product (`r16(0.5f * g * (1 + erf))`)."""
    I = in2d.shape[-1] // 2
    h, g = in2d[..., :I].to(F64), in2d[..., I:].to(F64)
    return h * bf16r(F.gelu(g, approximate="none"))


def geglu_autograd_din(in2d, dout):
    """float64 autograd of h * bf16(gelu(g)) with the rounding straight-through: d_h = dout * bf16(gelu(g)),
    d_g = dout * h * gelu'(g) (geglu_bwd_kernel)."""
    x = in2d.to(F64).detach().requires_grad_(True)
    I = x.shape[-1] // 2
    out = x[..., :I] * bf16_st(F.gelu(x[..., I:], approximate="none"))
    (out * dout.to(F64)).sum().backward()
    return x.grad


# ------------------------------------------------------------------------------------------------ spatial movers (NHWC)
def upsample2x_ref(x_nhwc):
    y = F.interpolate(x_nhwc.permute(0, 3, 1, 2).to(F64), scale_factor=2, mode="nearest")
    return y.permute(0, 2, 3, 1)


def upsample2x_bwd_ref(dy_nhwc):
    """Adjoint of the nearest 2x upsample: each input pixel receives the sum of its four children."""
    N, H2, W2, C = dy_nhwc.shape
    return dy_nhwc.to(F64).reshape(N, H2 // 2, 2, W2 // 2, 2, C).sum(dim=(2, 4))


def im2col_s2_ref(x_nhwc, pad):
    """Rows [N * H/2 * W/2, 9 * C] of the stride-2 3x3 conv, k = (r, s, c).  pad 1: symmetric padding 1 (UNet Downsample2D);
    pad 0: F.pad (0, 1, 0, 1) then no padding (VAE Downsample2D)."""
    N, H, W, C = x_nhwc.shape
    x = x_nhwc.permute(0, 3, 1, 2).to(F64)
    x = F.pad(x, (1, 1, 1, 1) if pad == 1 else (0, 1, 0, 1))
    cols = F.unfold(x, 3, stride=2)                                 # [N, C * 9, L], (c, r, s)
    L = cols.shape[-1]
    return cols.reshape(N, C, 9, L).permute(0, 3, 2, 1).reshape(N * L, 9 * C)


def col2im_s2_ref(dcols2d, N, H, W, C):
    """Adjoint of im2col_s2_ref(pad=1): F.fold of the (r, s, c) columns, padding stripped."""
    L = (H // 2) * (W // 2)
    cols = dcols2d.to(F64).reshape(N, L, 9, C).permute(0, 3, 2, 1).reshape(N, C * 9, L)
    x = F.fold(cols, (H + 2, W + 2), 3, stride=2)
    return x[:, :, 1:H + 1, 1:W + 1].permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------------ conv_in / conv_out
def conv_in_ref(latents_nchw, weight, bias, batch_out):
    """Conv2d(3x3, pad 1) on bf16-rounded fp32 NCHW latents and bf16 weights -> NHWC; output image n reads latents[n % Bsrc]."""
    Bs = latents_nchw.shape[0]
    x = bf16r(latents_nchw.to(F64))[torch.arange(batch_out) % Bs]
    y = F.conv2d(x, weight.to(F64), bias.to(F64), padding=1)
    return y.permute(0, 2, 3, 1)


def conv_out_ref(x_nhwc, weight, bias):
    """Conv2d(3x3, pad 1) NHWC bf16 -> NCHW, float64 before the kernels' single rounding to bf16."""
    return F.conv2d(x_nhwc.permute(0, 3, 1, 2).to(F64), weight.to(F64), bias.to(F64), padding=1)


def conv_out_bwd_ref(dy_nchw, weight):
    """d(conv_out)/dx: conv_transpose2d of the fp32 NCHW gradient with the bf16 weights -> NHWC."""
    return F.conv_transpose2d(dy_nchw.to(F64), weight.to(F64), padding=1).permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------------ time embedding / sampler
def timestep_embedding_ref(t, dim):
    """Timesteps(dim, flip_sin_to_cos=True, shift 0) in float64: [cos(t f_k) | sin(t f_k)], f_k = exp(-ln(1e4) k / half)."""
    half = dim // 2
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=F64) / half)
    arg = t.to(F64)[:, None] * f[None, :]
    return torch.cat([torch.cos(arg), torch.sin(arg)], dim=-1), f


def sampler_step_ref(eps, latents, coef_row, guidance, use_cfg, mode, noise=None):
    """float64 restatement of one sampler_step_ update with the coefficient row {sqrt(a_t), sqrt(1-a_t), c_x0, c_eps|c_xt, sigma}:
    CFG combine over [uncond | cond] then DDIM (mode 0) or DDPM (mode 1) — oracle/unet_oracle.ddim_step / ddpm_step."""
    c = coef_row.to(F64)
    n = latents.numel()
    e = eps.to(F64).reshape(-1)
    e = e[:n] + guidance * (e[n:] - e[:n]) if use_cfg else e[:n]
    xt = latents.to(F64).reshape(-1)
    x0 = (xt - c[1] * e) / c[0]
    if mode == 0:
        out = c[2] * x0 + c[3] * e
    else:
        out = c[2] * x0 + c[3] * xt + (c[4] * noise.to(F64).reshape(-1) if noise is not None else 0.0)
    return out.reshape(latents.shape)


# ------------------------------------------------------------------------------------------------ VAE helpers
def softmax_rows_ref(x2d, scale):
    return torch.softmax(x2d.to(F64) * scale, dim=-1)


def vae_sample_ref(h_nchw, wq, bq, z, scaling, round_mean=bf16r, round_logvar=bf16r):
    """quant_conv (1x1) + DiagonalGaussianDistribution.sample() * scaling, rounded where vae_sample_kernel rounds:
    mean = bf16(Wq h + b), logvar = clamp(bf16(Wq h + b), -30, 20); out = (mean + exp(logvar / 2) z) * scaling.
    `round_mean` / `round_logvar` replace the two roundings (e.g. by `neighbour_rounding`)."""
    L = h_nchw.shape[1] // 2
    m = torch.einsum("oc,nchw->nohw", wq.to(F64).reshape(2 * L, 2 * L), h_nchw.to(F64)) + bq.to(F64)[None, :, None, None]
    mean = round_mean(m[:, :L])
    logvar = round_logvar(m[:, L:]).clamp(-30.0, 20.0)
    return (mean + torch.exp(0.5 * logvar) * z.to(F64)) * scaling


# ------------------------------------------------------------------------------------------------ diffusion loss plumbing
def add_noise_ref(x0, noise, t, ac):
    a = ac.to(F64)[t.long()].view(-1, *([1] * (x0.dim() - 1)))
    return a.sqrt() * x0.to(F64) + (1 - a).sqrt() * noise.to(F64)


def mse_ref(pred, target):
    d = pred.to(F64) - target.to(F64)
    return (d * d).mean(), 2.0 * d / d.numel()


def mse_minsnr_ref(pred, target, t, ac, gamma):
    a = ac.to(F64)[t.long()]
    snr = a / (1 - a)
    w = snr.clamp(max=gamma) / snr
    d = pred.to(F64) - target.to(F64)
    wv = w.view(-1, *([1] * (d.dim() - 1)))
    return (wv * d * d).mean(), 2.0 * wv * d / d.numel()


# ------------------------------------------------------------------------------------------------ CLIP / splice helpers
def clip_patchify_ref(images, patch, kpad):
    """[N, 3, R, R] -> [N * G * G, kpad] unfolded patches in the conv weight's flatten order (c, ky, kx), zero padded."""
    N, C, R, _ = images.shape
    G = R // patch
    p = images.reshape(N, C, G, patch, G, patch).permute(0, 2, 4, 1, 3, 5).reshape(N * G * G, C * patch * patch)
    return F.pad(p, (0, kpad - C * patch * patch))


def segment_sum_rows_ref(src2d, seg, rows):
    Q = seg.numel() - 1
    out = torch.zeros(Q, src2d.shape[1], dtype=F64)
    s = src2d.to(F64)
    for q in range(Q):
        idx = rows[int(seg[q]):int(seg[q + 1])].long()
        if idx.numel():
            out[q] = s[idx].sum(0)
    return out

"""The float64 references of tests/test_tower_kernels_gpu.py (oracle/tower_kernels_oracle.py) against independent torch
formulations, torch.autograd and oracle/unet_oracle.py, on small shapes: a wrong reference must not let a wrong kernel pass."""
import math

import pytest
import torch
import torch.nn.functional as F

from dreamllm_b200.unet import scheduler_tables
from oracle import tower_kernels_oracle as R
from oracle import unet_oracle as UO

BF = torch.bfloat16
F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _vjp(fn, x, g):
    x = x.detach().to(F64).requires_grad_(True)
    (fn(x) * g).sum().backward()
    return x.grad


def test_ulp_diff_and_neighbour_rounding():
    one = torch.tensor([1.0], dtype=BF)
    nxt = torch.nextafter(one.float(), torch.tensor([2.0])).to(BF)        # rounds to 1: fp32 step is below bf16's
    assert int(R.ulp_diff(one, nxt)) == 0
    up = torch.tensor([1.0 + 2.0 ** -7], dtype=BF)                        # bf16 spacing at 1 is 2^-7
    assert int(R.ulp_diff(one, up)) == 1
    assert int(R.ulp_diff(torch.tensor([0.0], dtype=BF), torch.tensor([-0.0], dtype=BF))) == 0
    tiny = torch.tensor([2.0 ** -133], dtype=BF)                          # smallest positive bf16 (subnormal)
    assert int(R.ulp_diff(tiny, -tiny)) == 2
    assert int(R.ulp_diff(torch.tensor([-1.0], dtype=BF), torch.tensor([-1.0 - 2.0 ** -7], dtype=BF))) == 1
    # a value on a rounding midpoint may round to either neighbour; one far from it has a single answer
    mid = torch.tensor([1.0 + 2.0 ** -8, -(1.0 + 2.0 ** -8), 1.0 + 2.0 ** -9], dtype=F64)
    other = R.neighbour_rounding(mid)
    near = R.bf16r(mid)
    assert other[0] != near[0] and other[1] != near[1] and other[2] == near[2]
    assert {float(other[0]), float(near[0])} == {1.0, 1.0 + 2.0 ** -7}
    assert {float(other[1]), float(near[1])} == {-1.0, -1.0 - 2.0 ** -7}


@pytest.mark.parametrize("C,G,silu", [(40, 4, True), (24, 2, False), (16, 4, True)])
def test_groupnorm_ref_vs_nn_groupnorm(C, G, silu):
    N, H, W = 2, 5, 3
    x = (3.0 + torch.randn(N, H, W, C, generator=_g(1))).to(BF)
    w = (1 + 0.3 * torch.randn(C, generator=_g(2))).to(BF)
    b = (0.2 * torch.randn(C, generator=_g(3))).to(BF)
    gn = torch.nn.GroupNorm(G, C, eps=1e-5).to(F64)
    with torch.no_grad():
        gn.weight.copy_(w.to(F64))
        gn.bias.copy_(b.to(F64))
        pre = gn(x.permute(0, 3, 1, 2).to(F64)).permute(0, 2, 3, 1)
    torch.testing.assert_close(R.groupnorm_pre(x, w, b, G, 1e-5), pre, rtol=1e-12, atol=1e-12)
    want = R.bf16r(pre)
    if silu:
        want = torch.nn.SiLU()(want)
    assert torch.equal(R.groupnorm_silu_ref(x, w, b, G, 1e-5, silu), want)
    var, mean = torch.var_mean(x.to(F64).reshape(N, H * W, G, C // G).permute(0, 2, 1, 3).reshape(N, G, -1), dim=-1, correction=0)
    m, rstd = R.groupnorm_stats(x, G, 1e-5)
    torch.testing.assert_close(m, mean, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(rstd, (var + 1e-5) ** -0.5, rtol=1e-12, atol=0)


@pytest.mark.parametrize("silu,dres", [(True, True), (False, False), (True, False)])
def test_groupnorm_autograd_dx_vs_closed_form(silu, dres):
    """The autograd reference equals the closed form groupnorm_bwd_nhwc evaluates: g = dy * silu'(y) * w,
    dx = rstd * (g - mean_g(g) - xhat * mean_g(g * xhat)) (+ dres), y = bf16(xhat * w + b)."""
    N, HW, C, G = 2, 12, 40, 4
    x = torch.randn(N, HW, C, generator=_g(4)).to(BF)
    w = (1 + 0.3 * torch.randn(C, generator=_g(5))).to(BF)
    b = (0.2 * torch.randn(C, generator=_g(6))).to(BF)
    dy = torch.randn(N, HW, C, generator=_g(7)).to(BF)
    dr = torch.randn(N, HW, C, generator=_g(8)).to(BF) if dres else None
    got = R.groupnorm_silu_autograd_dx(x, w, b, G, 1e-5, silu, dy, dr)
    mean, rstd = R.groupnorm_stats(x, G, 1e-5)
    xg = x.to(F64).reshape(N, HW, G, C // G)
    xh = (xg - mean[:, None, :, None]) * rstd[:, None, :, None]
    y = R.bf16r(xh * w.to(F64).reshape(G, C // G) + b.to(F64).reshape(G, C // G))
    g = dy.to(F64).reshape(N, HW, G, C // G)
    if silu:
        s = torch.sigmoid(y)
        g = g * s * (1 + y * (1 - s))
    g = g * w.to(F64).reshape(G, C // G)
    m1 = g.mean(dim=(1, 3), keepdim=True)
    m2 = (g * xh).mean(dim=(1, 3), keepdim=True)
    want = (rstd[:, None, :, None] * (g - m1 - xh * m2)).reshape(N, HW, C)
    if dres:
        want = want + dr.to(F64)
    torch.testing.assert_close(got, want, rtol=1e-10, atol=1e-10)


def test_layernorm_refs_vs_closed_form():
    T, H = 9, 48
    x = (2 + torch.randn(T, H, generator=_g(9))).to(BF)
    w = (1 + 0.3 * torch.randn(H, generator=_g(10))).to(BF)
    b = (0.2 * torch.randn(H, generator=_g(11))).to(BF)
    dy = torch.randn(T, H, generator=_g(12)).to(BF)
    dr = torch.randn(T, H, generator=_g(13)).to(BF)
    x64 = x.to(F64)
    mean = x64.mean(-1, keepdim=True)
    rstd = ((x64 - mean) ** 2).mean(-1, keepdim=True).add(1e-5).rsqrt()
    xh = (x64 - mean) * rstd
    torch.testing.assert_close(R.layernorm_ref(x, w, b, 1e-5), xh * w.to(F64) + b.to(F64), rtol=1e-12, atol=1e-12)
    g = dy.to(F64) * w.to(F64)
    want = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True)) + dr.to(F64)
    torch.testing.assert_close(R.layernorm_autograd_dx(x, w, b, 1e-5, dy, dr), want, rtol=1e-10, atol=1e-10)


def test_geglu_refs_vs_closed_form():
    T, I = 7, 24
    x = (1.5 * torch.randn(T, 2 * I, generator=_g(14))).to(BF)
    d = torch.randn(T, I, generator=_g(15)).to(BF)
    h, g = x[:, :I].to(F64), x[:, I:].to(F64)
    cdf = 0.5 * (1 + torch.erf(g / math.sqrt(2)))
    pdf = torch.exp(-0.5 * g * g) / math.sqrt(2 * math.pi)
    gelu_b = R.bf16r(g * cdf)
    assert torch.equal(R.geglu_ref(x), h * gelu_b)
    want = torch.cat([d.to(F64) * gelu_b, d.to(F64) * h * (cdf + g * pdf)], dim=1)
    torch.testing.assert_close(R.geglu_autograd_din(x, d), want, rtol=1e-12, atol=1e-12)


def test_movers_refs_vs_indexing_and_autograd():
    N, H, W, C = 2, 6, 10, 3
    x = torch.randn(N, H, W, C, generator=_g(16), dtype=F64)
    up = R.upsample2x_ref(x)
    assert torch.equal(up, x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))
    gu = torch.randn(up.shape, generator=_g(17), dtype=F64)
    torch.testing.assert_close(R.upsample2x_bwd_ref(gu), _vjp(R.upsample2x_ref, x, gu), rtol=1e-12, atol=1e-12)
    # im2col rows against the stride-2 conv they feed (both paddings), and col2im as the autograd adjoint of pad 1
    wconv = torch.randn(5, C, 3, 3, generator=_g(18), dtype=F64)
    wk = wconv.permute(0, 2, 3, 1).reshape(5, 9 * C)                          # k = (r, s, c)
    for pad in (1, 0):
        cols = R.im2col_s2_ref(x, pad)
        xp = F.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1) if pad == 1 else (0, 1, 0, 1))
        y = F.conv2d(xp, wconv, stride=2).permute(0, 2, 3, 1).reshape(-1, 5)
        torch.testing.assert_close(cols @ wk.T, y, rtol=1e-12, atol=1e-12)
        # explicit (h, w, tap) indexing for a few rows
        for row in (0, 7, cols.shape[0] - 1):
            n, rem = divmod(row, (H // 2) * (W // 2))
            ho, wo = divmod(rem, W // 2)
            for tap in range(9):
                hh, ww = 2 * ho + tap // 3 - pad, 2 * wo + tap % 3 - pad
                v = x[n, hh, ww] if 0 <= hh < H and 0 <= ww < W else torch.zeros(C, dtype=F64)
                assert torch.equal(cols[row, tap * C:(tap + 1) * C], v)
    gc = torch.randn(N * (H // 2) * (W // 2), 9 * C, generator=_g(19), dtype=F64)
    torch.testing.assert_close(R.col2im_s2_ref(gc, N, H, W, C), _vjp(lambda t: R.im2col_s2_ref(t, 1), x, gc), rtol=1e-12, atol=1e-12)


def test_conv_refs_vs_autograd_and_modules():
    B, C, H, W = 2, 16, 5, 7
    x = torch.randn(B, H, W, C, generator=_g(20)).to(BF)
    w = (0.1 * torch.randn(4, C, 3, 3, generator=_g(21))).to(BF)
    b = (0.1 * torch.randn(4, generator=_g(22))).to(BF)
    conv = torch.nn.Conv2d(C, 4, 3, padding=1).to(F64)
    with torch.no_grad():
        conv.weight.copy_(w.to(F64))
        conv.bias.copy_(b.to(F64))
        want = conv(x.permute(0, 3, 1, 2).to(F64))
    torch.testing.assert_close(R.conv_out_ref(x, w, b), want, rtol=1e-12, atol=1e-12)
    dy = torch.randn(B, 4, H, W, generator=_g(23))
    torch.testing.assert_close(R.conv_out_bwd_ref(dy, w), _vjp(lambda t: R.conv_out_ref(t, w, b), x, dy.to(F64)),
                               rtol=1e-12, atol=1e-12)
    # conv_in: bf16-rounded fp32 latents; CFG batch reads latents[n % Bsrc]
    lat = torch.randn(B, 4, H, W, generator=_g(24))
    wi = (0.1 * torch.randn(8, 4, 3, 3, generator=_g(25))).to(BF)
    bi = (0.1 * torch.randn(8, generator=_g(26))).to(BF)
    got = R.conv_in_ref(lat, wi, bi, 2 * B)
    one = F.conv2d(lat.to(BF).to(F64), wi.to(F64), bi.to(F64), padding=1).permute(0, 2, 3, 1)
    assert torch.equal(got, torch.cat([one, one]))


def test_timestep_embedding_ref_vs_unet_oracle():
    t = torch.tensor([0, 1, 999, 500])
    for dim in (320, 256):
        want = UO.timestep_embedding(t, dim)                                  # fp32: argument error up to ~999 * 2^-24 * few
        got, f = R.timestep_embedding_ref(t, dim)
        assert got.shape == (4, dim) and f.shape == (dim // 2,)
        torch.testing.assert_close(got, want.to(F64), rtol=0, atol=5e-4)
        assert torch.equal(got[0], torch.cat([torch.ones(dim // 2, dtype=F64), torch.zeros(dim // 2, dtype=F64)]))


@pytest.mark.parametrize("kind", ["ddim", "ddpm"])
@pytest.mark.parametrize("use_cfg", [True, False])
def test_sampler_restatement_vs_unet_oracle(kind, use_cfg):
    n_steps, guidance = 20, 7.5
    ts, coef = scheduler_tables(n_steps, kind)
    ac = UO.alphas_cumprod().to(F64)
    ratio = 1000 // n_steps
    g = _g(27)
    x = torch.randn(2, 4, 6, 6, generator=g, dtype=F64)
    for i in (0, 1, n_steps - 1):
        t = int(ts[i])
        eu, ec, z = (torch.randn(2, 4, 6, 6, generator=g, dtype=F64) for _ in range(3))
        e = UO.cfg_combine(eu, ec, guidance) if use_cfg else eu
        eps = torch.cat([eu, ec]) if use_cfg else eu
        mode = 0 if kind == "ddim" else 1
        got = R.sampler_step_ref(eps, x, coef[i], guidance, use_cfg, mode, noise=z if mode else None)
        want = UO.ddim_step(x, e, t, ratio, ac) if mode == 0 else UO.ddpm_step(x, e, t, ratio, ac, z)
        torch.testing.assert_close(got, want, rtol=2e-5, atol=2e-5 * float(want.abs().max()))


def test_vae_sample_softmax_and_loss_refs():
    B, L, H, W = 2, 4, 3, 5
    h = torch.randn(B, 2 * L, H, W, generator=_g(28))
    wq = (0.3 * torch.randn(2 * L, 2 * L, generator=_g(29))).to(BF)
    bq = torch.tensor([0, 0, 0, 0, 50.0, -60.0, 0, 0]).to(BF)                  # logvar of channel 0 past +20, channel 1 past -30
    z = torch.randn(B, L, H, W, generator=_g(30))
    m = F.conv2d(h.to(F64), wq.to(F64).view(2 * L, 2 * L, 1, 1), bq.to(F64))
    mean, logvar = m[:, :L].float().to(BF).to(F64), m[:, L:].float().to(BF).to(F64)
    std = torch.exp(0.5 * torch.clamp(logvar, -30, 20))
    got = R.vae_sample_ref(h, wq, bq, z, 0.18215)
    torch.testing.assert_close(got, (mean + std * z.to(F64)) * 0.18215, rtol=1e-12, atol=1e-12)
    assert float(std[:, 0].max()) == math.exp(10.0) and float(std[:, 1].max()) == math.exp(-15.0)
    x = torch.randn(5, 24, generator=_g(31))
    torch.testing.assert_close(R.softmax_rows_ref(x, 0.3), F.softmax(0.3 * x.to(F64), dim=-1), rtol=1e-12, atol=1e-15)
    # losses: autograd of the float64 loss gives the reference dpred
    ac = UO.alphas_cumprod()
    t = torch.tensor([10, 900])
    p, tg = torch.randn(2, 4, 3, 3, generator=_g(32)), torch.randn(2, 4, 3, 3, generator=_g(33))
    loss, dp = R.mse_ref(p, tg)
    torch.testing.assert_close(loss, F.mse_loss(p.to(F64), tg.to(F64)), rtol=1e-12, atol=0)
    torch.testing.assert_close(dp, _vjp(lambda q: F.mse_loss(q, tg.to(F64)), p, torch.tensor(1.0, dtype=F64)), rtol=1e-12, atol=0)
    a = ac[t].to(F64)
    snr = a / (1 - a)
    wv = torch.minimum(snr, torch.tensor(5.0, dtype=F64)) / snr
    loss2, dp2 = R.mse_minsnr_ref(p, tg, t, ac, 5.0)
    per = ((p.to(F64) - tg.to(F64)) ** 2).mean(dim=(1, 2, 3))
    torch.testing.assert_close(loss2, (per * wv).mean(), rtol=1e-12, atol=0)
    fn = lambda q: (((q - tg.to(F64)) ** 2).mean(dim=(1, 2, 3)) * wv).mean()  # noqa: E731
    torch.testing.assert_close(dp2, _vjp(fn, p, torch.tensor(1.0, dtype=F64)), rtol=1e-12, atol=0)
    x0, nz = torch.randn(2, 4, 3, 3, generator=_g(34)), torch.randn(2, 4, 3, 3, generator=_g(35))
    torch.testing.assert_close(R.add_noise_ref(x0, nz, t, ac), UO.add_noise(x0, nz, t, ac).to(F64), rtol=1e-6, atol=1e-6)


def test_clip_refs_vs_conv_and_loops():
    N, R_, p = 2, 28, 14
    img = torch.randn(N, 3, R_, R_, generator=_g(36), dtype=F64)
    w = torch.randn(6, 3, p, p, generator=_g(37), dtype=F64)
    cols = R.clip_patchify_ref(img, p, 600)
    assert cols.shape == (N * 4, 600) and torch.equal(cols[:, 3 * p * p:], torch.zeros(N * 4, 600 - 3 * p * p, dtype=F64))
    conv = F.conv2d(img, w, stride=p).permute(0, 2, 3, 1).reshape(N * 4, 6)
    torch.testing.assert_close(cols[:, :3 * p * p] @ w.reshape(6, -1).T, conv, rtol=1e-12, atol=1e-12)
    src = torch.randn(10, 16, generator=_g(38), dtype=F64)
    seg = torch.tensor([0, 3, 3, 7])
    rows = torch.tensor([1, 1, 9, 0, 2, 2, 5])
    got = R.segment_sum_rows_ref(src, seg, rows)
    want = torch.stack([src[1] + src[1] + src[9], torch.zeros(16, dtype=F64), src[0] + src[2] + src[2] + src[5]])
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)

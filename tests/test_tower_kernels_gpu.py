"""UNet / VAE / CLIP HBM-bound kernels, one launch at a time, against float64 references (oracle/tower_kernels_oracle.py).

Inputs are seeded on the host (the GEGLU grid-fold test draws its 5 GB input on the device from a seeded generator).  Where a kernel
rounds to bf16 mid-formula, the reference rounds at the same point.  The shapes are the ones the kernels branch on: GroupNorm at the
production group sizes (an 8-channel vector straddling two groups, or holding several), the LayerNorm warp variants and the
CTA-per-row kernel, the GEGLU grid fold, the conv_out direct fallback, the device-side step counters.

bf16 criterion (`_close_bf16`): every element within 1 bf16 ulp of the reference rounded once, and at most 1 % of the elements
differing from it at all.  A kernel computes the pre-rounding value in fp32, so near a rounding midpoint it may land on the other
bf16 neighbour; where the kernel rounds an intermediate and then applies a steep function (SiLU's negative tail), that other
neighbour is passed as `alt`.  Where a value cancels to near zero, the fp32 error of the terms (`atol`) can exceed an ulp of the
result; it is derived per test from the magnitudes of the terms.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import tower_kernels_oracle as R

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
F64 = torch.float64
EPS = 1e-5


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _ops():
    from dreamllm_b200 import ops
    return ops


def _close_bf16(got, ref, atol=0.0, alt=None, max_frac=1e-2, what=""):
    got = got.cpu()
    want = ref.to(torch.float32).to(BF)
    d0 = R.ulp_diff(got, want)
    d = d0 if alt is None else torch.minimum(d0, R.ulp_diff(got, alt.to(torch.float32).to(BF)))
    err = (got.to(F64) - ref).abs()
    bad = (d > 1) & (err > atol + 2.0 ** -8 * ref.abs())
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements off by more than 1 ulp (worst {int(d.max())} ulp); "
                             f"first at flat index {i}: got {float(got.flatten()[i])}, reference {float(ref.flatten()[i])}")
    frac = float((d0 > 0).double().mean())
    assert frac <= max_frac, f"{what}: {frac:.4f} of the elements differ from the reference rounding (at most {max_frac} allowed)"


# ------------------------------------------------------------------------------------------------ GroupNorm (+SiLU)
G = 32
# (C, HW, N): channels per group 10, 20, 30, 40, 60, 80 (SD-2.1 / SDXL widths and decoder concats: vectors straddle groups),
# 4 (VAE 128: several groups per vector) and 16; planes 8^2 / 16^2 / 64^2 walk gn_rows' halving, 256^2 its >128-chunk doubling
GN_SHAPES = [(320, 64 * 64, 2), (640, 16 * 16, 3), (960, 8 * 8, 3), (1280, 8 * 8, 2), (1920, 16 * 16, 1), (2560, 8 * 8, 2),
             (128, 256 * 256, 1), (512, 64 * 64, 1)]


def _gn_inputs(C, HW, N, offset, seed):
    cpg = C // G
    sign = 1.0 - 2.0 * ((torch.arange(C) // cpg) % 2).double()                # groups alternate +offset / -offset
    x = (offset * sign + torch.randn(N, HW, C, generator=_g(seed), dtype=F64)).to(BF)
    w = (1 + 0.3 * torch.randn(C, generator=_g(seed + 1))).to(BF)
    b = (0.3 * torch.randn(C, generator=_g(seed + 2))).to(BF)
    return x, w, b


def _check_groupnorm_fwd(C, HW, N, silu, offset, seed):
    ops = _ops()
    x, w, b = _gn_inputs(C, HW, N, offset, seed)
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    y1 = ops.groupnorm(xd, wd, bd, G, EPS, silu)
    y2, st = ops.groupnorm(xd, wd, bd, G, EPS, silu, return_stats=True)
    assert torch.equal(y1, y2), "fused and stats+apply GroupNorm differ"
    # statistics: fp32 sums of bf16 values; a stable reduction keeps the mean within 1e-5 of the group's std (plus the fp32
    # resolution of the mean itself) and rstd within 1e-4 relative — 1/40 of a bf16 ulp of the normalised output
    mean64, rstd64 = R.groupnorm_stats(x, G, EPS)
    st = st.cpu().to(F64)
    merr = ((st[..., 0] - mean64).abs() / (1e-5 / rstd64 + 2.0 ** -22 * mean64.abs())).max()
    rerr = (st[..., 1] / rstd64 - 1).abs().max()
    assert merr <= 1 and rerr <= 1e-4, f"GroupNorm stats: mean error {float(merr):.3g} of its bound, rstd relative error {float(rerr):.3g}"
    # fp32 (x - mean) * rstd * w + b: a few fp32 ulps of each term, the fp32 mean's error scaled by rstd * w
    mc, rc = (s.repeat_interleave(C // G, dim=1)[:, None] for s in (mean64, rstd64))
    w64 = w.to(F64)
    atol = 2.0 ** -19 * (((x.to(F64) - mc) * rc * w64).abs() + b.to(F64).abs() + w64.abs() * (1 + rc * mc.abs()))
    pre = R.groupnorm_pre(x, w, b, G, EPS)
    t, t_alt = R.bf16r(pre), R.neighbour_rounding(pre, atol=atol)
    ref, alt = (F.silu(t), F.silu(t_alt)) if silu else (t, t_alt)
    _close_bf16(y1, ref, atol=atol, alt=alt, what=f"groupnorm C={C} HW={HW} N={N} silu={silu} offset={offset}")


@pytest.mark.parametrize("silu", [True, False])
@pytest.mark.parametrize("C,HW,N", GN_SHAPES)
def test_groupnorm_fwd_vs_float64(C, HW, N, silu):
    _check_groupnorm_fwd(C, HW, N, silu, 0.0, seed=C + HW + N)


@pytest.mark.parametrize("offset", [0.0, 16.0, 64.0, 128.0])
@pytest.mark.parametrize("C,HW", [(320, 64 * 64), (128, 256 * 256)])
def test_groupnorm_fwd_large_mean_over_std(C, HW, offset):
    """Inputs whose mean is 16 to 128 standard deviations from zero: the variance must not come from E[x^2] - mean^2."""
    _check_groupnorm_fwd(C, HW, 1, True, offset, seed=7 + C)


GN_BWD_SHAPES = [(320, 16 * 16, 2), (640, 8 * 8, 3), (960, 8 * 8, 1), (1280, 8 * 8, 1), (1920, 8 * 8, 1), (2560, 8 * 8, 1),
                 (128, 64 * 64, 1), (512, 16 * 16, 2)]


@pytest.mark.parametrize("silu,dres", [(True, True), (True, False), (False, True), (False, False)])
@pytest.mark.parametrize("C,HW,N", GN_BWD_SHAPES)
def test_groupnorm_bwd_vs_float64_autograd(C, HW, N, silu, dres):
    ops = _ops()
    x, w, b = _gn_inputs(C, HW, N, 8.0, seed=3 * C + HW)
    dy = torch.randn(N, HW, C, generator=_g(C + 5)).to(BF)
    dr = torch.randn(N, HW, C, generator=_g(C + 6)).to(BF) if dres else None
    _, st = ops.groupnorm(x.cuda(), w.cuda(), b.cuda(), G, EPS, silu, return_stats=True)
    dx = ops.groupnorm_bwd(dy.cuda(), x.cuda(), w.cuda(), b.cuda(), st, G, silu, dres=dr.cuda() if dres else None).cpu().to(F64)
    ref = R.groupnorm_silu_autograd_dx(x, w, b, G, EPS, silu, dy, dr)
    # per group: the bf16 output rounding alone gives |err| <= 2^-8 |ref| elementwise, i.e. ||err||_2 <= 2^-8 ||ref||_2
    err = (dx - ref).reshape(N, HW, G, C // G).transpose(1, 2).reshape(N, G, -1)
    refg = ref.reshape(N, HW, G, C // G).transpose(1, 2).reshape(N, G, -1)
    rel2 = err.norm(dim=-1) / refg.norm(dim=-1)
    relinf = err.abs().amax(-1) / refg.abs().amax(-1)
    assert float(rel2.max()) <= 2.0 ** -8 and float(relinf.max()) <= 2.0 ** -7, \
        f"groupnorm_bwd: per-group ||err||/||ref|| {float(rel2.max()):.3g} (2-norm), {float(relinf.max()):.3g} (max)"


# ------------------------------------------------------------------------------------------------ LayerNorm
# warp kernels: VPL 2 up to H = 512 (64 vectors), VPL 4 up to 1024, VPL 6 up to 1536; CTA-per-row kernel above
LN_H_WARP = [320, 512, 520, 1024, 1032, 1280, 1536]
LN_H_CTA = [1544, 2048, 4096]


@pytest.mark.parametrize("H", LN_H_WARP + LN_H_CTA)
def test_layernorm_fwd_vs_float64(H):
    ops = _ops()
    T = 37                                                                   # not a multiple of the 8 row-warps per CTA
    x = (1.5 + 2 * torch.randn(T, H, generator=_g(H))).to(BF)
    w = (1 + 0.3 * torch.randn(H, generator=_g(H + 1))).to(BF)
    b = (0.3 * torch.randn(H, generator=_g(H + 2))).to(BF)
    y = ops.layernorm_fwd(x.cuda(), w.cuda(), b.cuda(), EPS)
    ref = R.layernorm_ref(x, w, b, EPS)
    # fp32 (x - mean) * rstd * w + b: a few fp32 ulps of each term, the fp32 mean's error scaled by rstd * w
    m64 = x.to(F64).mean(-1, keepdim=True)
    r64 = (x.to(F64).var(-1, correction=0, keepdim=True) + EPS).rsqrt()
    atol = 2.0 ** -19 * ((ref - b.to(F64)).abs() + b.to(F64).abs() + w.to(F64).abs() * (1 + r64 * m64.abs()))
    _close_bf16(y, ref, atol=atol, what=f"layernorm_fwd H={H}")


@pytest.mark.parametrize("dres", [True, False])
@pytest.mark.parametrize("H", LN_H_WARP)
def test_layernorm_bwd_vs_float64_autograd(H, dres):
    ops = _ops()
    T = 37
    x = (0.5 + torch.randn(T, H, generator=_g(2 * H))).to(BF)
    w = (1 + 0.3 * torch.randn(H, generator=_g(2 * H + 1))).to(BF)
    b = (0.3 * torch.randn(H, generator=_g(2 * H + 2))).to(BF)
    dy = torch.randn(T, H, generator=_g(2 * H + 3)).to(BF)
    dr = torch.randn(T, H, generator=_g(2 * H + 4)).to(BF) if dres else None
    dx = ops.layernorm_bwd(dy.cuda(), x.cuda(), w.cuda(), EPS, dres=dr.cuda() if dres else None).cpu().to(F64)
    ref = R.layernorm_autograd_dx(x, w, b, EPS, dy, dr)
    err = dx - ref
    rel2 = err.norm(dim=-1) / ref.norm(dim=-1)
    relinf = err.abs().amax(-1) / ref.abs().amax(-1)
    assert float(rel2.max()) <= 2.0 ** -8 and float(relinf.max()) <= 2.0 ** -7, \
        f"layernorm_bwd H={H}: per-row ||err||/||ref|| {float(rel2.max()):.3g} (2-norm), {float(relinf.max()):.3g} (max)"


# ------------------------------------------------------------------------------------------------ GEGLU
def _gelu_atol(g64):
    # the kernel's 0.5 g (1 + erff(g / sqrt 2)) in fp32: erff is good to a few ulps of 1, and for g < 0 the sum 1 + erff cancels, so
    # the error is a few fp32 ulps of |g| in absolute terms (up to 4e-5 of gelu(g) itself near g = -3)
    return 2.0 ** -21 * (1 + g64.abs())


def _gelu_alt(g64):
    return R.neighbour_rounding(F.gelu(g64, approximate="none"), atol=_gelu_atol(g64))


def _geglu_atol(h64, g64):
    return h64.abs() * _gelu_atol(g64)


@pytest.mark.parametrize("I", [1280, 2560, 5120])
def test_geglu_fwd_past_the_grid_fold(I):
    """T > 262 140 rows splits the launch (blockIdx.y <= 65535 row groups of 4): check the rows around the fold boundary, the first
    rows and the last rows of every T in 262 140 ... 262 150 against float64."""
    ops = _ops()
    Tmax, fold = 262150, 65535 * 4
    gen = torch.Generator(device="cuda").manual_seed(I)
    x = torch.randn(Tmax, 2 * I, device="cuda", generator=gen, dtype=BF).mul_(1.5)
    for T in range(fold, Tmax + 1):
        out = ops.geglu(x[:T])
        rows = torch.cat([torch.arange(0, 4), torch.arange(fold - 6, T)])
        xs = x[rows.cuda()].cpu()
        h64, g64 = xs[:, :I].to(F64), xs[:, I:].to(F64)
        ref = R.geglu_ref(xs)
        _close_bf16(out[rows.cuda()], ref, atol=_geglu_atol(h64, g64), alt=h64 * _gelu_alt(g64), what=f"geglu I={I} T={T}")
        del out


@pytest.mark.parametrize("I", [1280, 2560, 5120])
def test_geglu_bwd_vs_float64_autograd(I):
    ops = _ops()
    T = 301
    x = (1.5 * torch.randn(T, 2 * I, generator=_g(I + 9))).to(BF)
    d = torch.randn(T, I, generator=_g(I + 10)).to(BF)
    din = ops.geglu_bwd(d.cuda(), x.cuda()).cpu()
    ref = R.geglu_autograd_din(x, d)
    h64, g64, d64 = x[:, :I].to(F64), x[:, I:].to(F64), d.to(F64)
    # d_h = dout * bf16(gelu(g)): the product of two bf16 values is exact in fp32, so only the gelu rounding may differ
    _close_bf16(din[:, :I], ref[:, :I], atol=_geglu_atol(d64, g64), alt=d64 * _gelu_alt(g64), what=f"geglu_bwd d_h I={I}")
    # d_g = dout * h * (Phi(g) + g phi(g)) in fp32: cancels to zero near g = -0.75
    atol_g = (d64 * h64).abs() * 2.0 ** -20 * (1 + g64.abs())
    _close_bf16(din[:, I:], ref[:, I:], atol=atol_g, what=f"geglu_bwd d_g I={I}")


# ------------------------------------------------------------------------------------------------ spatial movers
def _adjoint_gap(fx, g, x, bg):
    """|<fwd(x), g> - <x, bwd(g)>| against the bf16 rounding of bwd(g)'s sums: sum |x| |bwd(g)| 2^-8."""
    lhs = (fx.to(F64) * g.to(F64)).sum()
    rhs = (x.to(F64) * bg.to(F64)).sum()
    return float((lhs - rhs).abs()), float((x.to(F64).abs() * bg.to(F64).abs()).sum()) * 2.0 ** -8


@pytest.mark.parametrize("C", [8, 40, 328])                                # 1, 5 and 41 channel vectors
def test_spatial_movers_bitexact_and_adjoint(C):
    ops = _ops()
    N = 2
    # nearest 2x upsample on a non-square plane with odd sides
    x = torch.randn(N, 5, 7, C, generator=_g(C)).to(BF)
    up = ops.upsample2x(x.cuda()).cpu()
    assert torch.equal(up, R.upsample2x_ref(x).to(BF))
    gu = torch.randn(up.shape, generator=_g(C + 1)).to(BF)
    dx = ops.upsample2x_bwd(gu.cuda()).cpu()
    _close_bf16(dx, R.upsample2x_bwd_ref(gu), what="upsample2x_bwd")
    gap, tol = _adjoint_gap(up, gu, x, dx)
    assert gap <= tol, ("upsample2x adjoint", gap, tol)
    # stride-2 im2col (pad 1 and pad 0) and the pad-1 col2im
    H, W = 6, 10
    x = torch.randn(N, H, W, C, generator=_g(C + 2)).to(BF)
    for pad in (1, 0):
        cols = ops.im2col_s2(x.cuda(), pad=pad).cpu()
        assert torch.equal(cols, R.im2col_s2_ref(x, pad).to(BF)), f"im2col_s2 pad={pad}"
    cols = ops.im2col_s2(x.cuda(), pad=1).cpu()
    gc = torch.randn(cols.shape, generator=_g(C + 3)).to(BF)
    dxc = ops.col2im_s2(gc.cuda(), N, H, W, C).cpu()
    _close_bf16(dxc, R.col2im_s2_ref(gc, N, H, W, C), what="col2im_s2")
    gap, tol = _adjoint_gap(cols, gc, x, dxc)
    assert gap <= tol, ("im2col_s2 / col2im_s2 adjoint", gap, tol)
    # channel concat / split / column copy
    Cb = 16
    a = torch.randn(N, H, W, C, generator=_g(C + 4)).to(BF)
    bb = torch.randn(N, H, W, Cb, generator=_g(C + 5)).to(BF)
    cat = ops.concat_channels(a.cuda(), bb.cuda())
    assert torch.equal(cat.cpu(), torch.cat([a, bb], dim=-1))
    s1, s2 = ops.split_channels(cat, C)
    assert torch.equal(s1.cpu(), a) and torch.equal(s2.cpu(), bb)
    s1, s2 = ops.split_channels(cat, 8)
    assert torch.equal(s1.cpu(), cat.cpu()[..., :8]) and torch.equal(s2.cpu(), cat.cpu()[..., 8:])
    dst = torch.randn(N * H * W, C + 24, generator=_g(C + 6)).to(BF)
    src = torch.randn(N * H * W, C, generator=_g(C + 7)).to(BF)
    got = ops.copy_cols_(src.cuda(), dst.cuda(), 16).cpu()
    want = dst.clone()
    want[:, 16:16 + C] = src
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ conv_in / conv_out
def _conv_bound(ref, abs_sum):
    """bf16 output rounding (<= 2^-8 |ref|) + fp32 accumulation (a few fp32 ulps of the sum of |terms|)."""
    return 2.0 ** -8 * ref.abs() + 2.0 ** -20 * abs_sum


# (Cin, Cout, Bsrc, batch_out, H, W): Cin 4 / 3 take im2col + GEMM, Cin >= 8 the direct kernel (Cin * 9 * Cout * 4 <= 96 KiB)
@pytest.mark.parametrize("Cin,Cout,Bsrc,batch_out,H,W", [(4, 320, 2, 4, 16, 24), (3, 128, 1, 1, 20, 12), (8, 64, 2, 4, 9, 13),
                                                         (16, 32, 1, 2, 8, 8)])
def test_conv_in_vs_float64(Cin, Cout, Bsrc, batch_out, H, W):
    ops = _ops()
    lat = torch.randn(Bsrc, Cin, H, W, generator=_g(Cin + Cout))
    w = (0.2 * torch.randn(Cout, Cin, 3, 3, generator=_g(Cin + Cout + 1))).to(BF)
    b = (0.2 * torch.randn(Cout, generator=_g(Cin + Cout + 2))).to(BF)
    y = ops.conv_in(lat.cuda(), w.cuda(), b.cuda(), batch_out).cpu().to(F64)
    ref = R.conv_in_ref(lat, w, b, batch_out)
    abs_sum = R.conv_in_ref(lat.abs(), w.abs(), b.abs(), batch_out)
    err = (y - ref).abs()
    assert bool((err <= _conv_bound(ref, abs_sum)).all()), f"conv_in: worst |err| / |ref|inf = {float(err.max() / ref.abs().max()):.3g}"


def test_conv_in_direct_rejects_cout_not_multiple_of_8():
    ops = _ops()
    lat = torch.randn(1, 4, 8, 8, generator=_g(40)).cuda()
    w = torch.zeros(12, 4, 3, 3, dtype=BF, device="cuda")
    with pytest.raises(RuntimeError, match="dllm_conv_in failed: invalid shape"):
        ops.conv_in(lat, w, torch.zeros(12, dtype=BF, device="cuda"), 1)


# (C, H, W, Cout): C % 64 == 0 with W tiling 128 takes the implicit GEMM; C = 96 or W = 96 / 168 the direct kernel
@pytest.mark.parametrize("C,H,W,Cout", [(320, 64, 64, 4), (320, 64, 64, 3), (320, 64, 64, 8), (320, 8, 96, 4), (320, 6, 168, 3),
                                        (320, 5, 168, 8), (96, 8, 64, 4), (96, 7, 96, 8)])
def test_conv_out_vs_float64(C, H, W, Cout):
    ops = _ops()
    x = torch.randn(1, H, W, C, generator=_g(C + W + Cout)).to(BF)
    w = (0.05 * torch.randn(Cout, C, 3, 3, generator=_g(C + W + Cout + 1))).to(BF)
    b = (0.2 * torch.randn(Cout, generator=_g(C + W + Cout + 2))).to(BF)
    y = ops.conv_out(x.cuda(), w.cuda(), b.cuda()).cpu().to(F64)
    ref = R.conv_out_ref(x, w, b)
    abs_sum = R.conv_out_ref(x.abs(), w.abs(), b.abs())
    err = (y - ref).abs()
    assert bool((err <= _conv_bound(ref, abs_sum)).all()), f"conv_out: worst |err| / |ref|inf = {float(err.max() / ref.abs().max()):.3g}"


@pytest.mark.parametrize("C,H,W", [(320, 16, 16), (320, 6, 168), (96, 9, 7)])
def test_conv_out_bwd_vs_float64(C, H, W):
    ops = _ops()
    dy = torch.randn(2, 4, H, W, generator=_g(C + H))
    w = (0.05 * torch.randn(4, C, 3, 3, generator=_g(C + H + 1))).to(BF)
    dx = ops.conv_out_bwd(dy.cuda(), w.cuda(), C).cpu().to(F64)
    ref = R.conv_out_bwd_ref(dy, w)
    abs_sum = R.conv_out_bwd_ref(dy.abs(), w.abs())
    err = (dx - ref).abs()
    assert bool((err <= _conv_bound(ref, abs_sum)).all()), f"conv_out_bwd: worst |err| / |ref|inf = {float(err.max() / ref.abs().max()):.3g}"


# ------------------------------------------------------------------------------------------------ time embedding / sampler
def _temb_bound(t, f, ref):
    """The kernel forms f = exp(-ln(1e4) k / half) and t * f in fp32 (fast-math exp2 of a rounded product): the argument carries up to
    2^-19 relative error (8.4 ulps of fp32), 1.9e-3 rad at t = 999, f = 1; cos/sin of the rounded argument add <= 2^-19 absolute.
    With the bf16 output rounding (<= 2^-8 relative): |err| <= 2^-8 (|ref| + delta) + delta, delta = 2^-19 (t f + 1)."""
    delta = 2.0 ** -19 * (t.to(F64)[:, None] * f[None, :] + 1)
    delta = torch.cat([delta, delta], dim=1)
    return 2.0 ** -8 * (ref.abs() + delta) + delta


@pytest.mark.parametrize("dim", [320, 256])
def test_timestep_embedding_vs_float64(dim):
    ops = _ops()
    sched = torch.tensor([999, 1, 0, 500, 981], dtype=torch.int32)
    B = 3
    for s in (0, 1, 2, 3):                                                   # the device-side step picks t = sched[step]
        out = ops.timestep_embedding(sched.cuda(), torch.tensor([s], dtype=torch.int32).cuda(), B, dim).cpu().to(F64)
        t = sched[s:s + 1].repeat(B)
        ref, f = R.timestep_embedding_ref(t, dim)
        err = (out - ref).abs()
        assert bool((err <= _temb_bound(t, f, ref)).all()), f"timestep_embedding step {s} (t={int(sched[s])}): max err {float(err.max()):.3g}"
    t = torch.tensor([0, 1, 999, 37], dtype=torch.int32)
    out = ops.timestep_embedding_batch(t.cuda(), dim).cpu().to(F64)
    ref, f = R.timestep_embedding_ref(t, dim)
    err = (out - ref).abs()
    assert bool((err <= _temb_bound(t, f, ref)).all()), f"timestep_embedding_batch: max err {float(err.max()):.3g}"


@pytest.mark.parametrize("use_cfg", [True, False])
@pytest.mark.parametrize("kind", ["ddim", "ddpm"])
def test_sampler_step_two_steps_vs_float64(kind, use_cfg):
    from dreamllm_b200.unet import scheduler_tables
    ops = _ops()
    n_steps, guidance, first = 20, 7.5, 3
    mode = 0 if kind == "ddim" else 1
    ts, coef = scheduler_tables(n_steps, kind)
    shape = (2, 4, 16, 16)
    n = math.prod(shape)
    lat = torch.randn(shape, generator=_g(50))
    noise = torch.randn(n_steps, n, generator=_g(51)) if mode else None
    step = torch.tensor([first], dtype=torch.int32).cuda()
    latd = lat.cuda()
    for i in (first, first + 1):
        eps = torch.randn((2 * shape[0] if use_cfg else shape[0], *shape[1:]), generator=_g(52 + i))
        before = latd.cpu()
        ops.sampler_step_(eps.cuda(), latd, coef.cuda(), step, guidance, use_cfg, mode, noise.cuda() if mode else None)
        got = latd.cpu().to(F64)
        ref = R.sampler_step_ref(eps, before, coef[i], guidance, use_cfg, mode, noise[i] if mode else None)
        # fp32 arithmetic: a few ulps of every term, the x0 terms amplified by 1/sqrt(a_t)
        c = coef[i].to(F64)
        e = eps.to(F64).reshape(-1)
        E = (e[:n].abs() + guidance * (e[n:].abs() + e[:n].abs())) if use_cfg else e.abs()
        xt = before.to(F64).reshape(-1).abs()
        mag = c[2].abs() / c[0] * (xt + c[1] * E) + (c[3].abs() * (E if mode == 0 else xt))
        if mode:
            mag = mag + c[4].abs() * noise[i].to(F64).abs()
        err = (got.reshape(-1) - ref.reshape(-1)).abs()
        assert bool((err <= 2.0 ** -20 * mag).all()), f"sampler {kind} cfg={use_cfg} step {i}: max err / bound {float((err / mag).max()):.3g}"
    assert int(step.item()) == first + 2, "the device step counter must advance once per call"


# ------------------------------------------------------------------------------------------------ VAE helpers
@pytest.mark.parametrize("cols", [8, 4096, 4104, 16384])
def test_softmax_rows_vs_float64(cols):
    ops = _ops()
    scale = 512 ** -0.5                                                      # the VAE mid-block attention: one head of C = 512
    g = _g(cols)
    rows = [30 * torch.randn(cols, generator=g),                              # ordinary scores
            500 * (2 * torch.rand(cols, generator=g) - 1),                    # large magnitude: exponents down to -44
            torch.full((cols,), 7.0),                                         # equal values: uniform 1 / cols
            torch.full((cols,), -1000.0),
            torch.where(torch.arange(cols) == cols // 3, 900.0, -300.0 * torch.rand(cols, generator=g))]
    x = torch.stack(rows).to(BF)
    got = ops.softmax_rows_(x.cuda().clone(), scale)
    _close_bf16(got, R.softmax_rows_ref(x, scale), max_frac=1.0, what=f"softmax_rows cols={cols}")


def test_vae_sample_vs_float64():
    ops = _ops()
    B, L, H, W = 2, 4, 16, 24
    h = torch.randn(B, 2 * L, H, W, generator=_g(60))
    wq = (0.3 * torch.randn(2 * L, 2 * L, generator=_g(61))).to(BF)
    bq = torch.tensor([0.1, -0.2, 0.3, 0.0, 45.0, -55.0, 0.5, -1.0]).to(BF)     # logvar 0 past +20, logvar 1 past -30
    z = torch.randn(B, L, H, W, generator=_g(62))
    got = ops.vae_sample(h.cuda(), wq.cuda(), bq.cuda(), z.cuda(), 0.18215).cpu().to(F64)
    refs = [R.vae_sample_ref(h, wq, bq, z, 0.18215, rm, rl) for rm in (R.bf16r, R.neighbour_rounding)
            for rl in (R.bf16r, R.neighbour_rounding)]
    # after the two bf16 roundings: fp32 mean + exp(logvar / 2) z (fast-math exp2 of a rounded argument: <= 2^-19 relative)
    m = refs[0] / 0.18215
    mean = R.vae_sample_ref(h, wq, bq, torch.zeros_like(z), 1.0)
    tol = 0.18215 * (2.0 ** -20 * mean.abs() + 2.0 ** -19 * (m - mean).abs()) + 1e-30
    ok = torch.zeros_like(got, dtype=torch.bool)
    for r in refs:
        ok |= (got - r).abs() <= tol
    assert bool(ok.all()), f"vae_sample: {int((~ok).sum())} elements off; max err {float((got - refs[0]).abs().max()):.3g}"
    assert float(got[:, 0].abs().max()) > 100 and float((got[:, 1] - 0.18215 * mean[:, 1]).abs().max()) < 1e-6   # the clamps bit


# ------------------------------------------------------------------------------------------------ diffusion loss plumbing
def test_add_noise_and_mse_losses_sdxl_size():
    """B = 16 SDXL latents (4 x 128 x 128): n = 1 048 576 through the single-CTA loss loops."""
    from oracle import unet_oracle as UO
    ops = _ops()
    B, shape = 16, (4, 128, 128)
    g = _g(70)
    x0, nz, pred, tgt = (torch.randn(B, *shape, generator=g) for _ in range(4))
    t = torch.randint(0, 1000, (B,), generator=g, dtype=torch.int32)
    ac = UO.alphas_cumprod()
    noisy = ops.add_noise(x0.cuda(), nz.cuda(), t.cuda(), ac.cuda()).cpu().to(F64)
    a = ac.to(F64)[t.long()].view(B, 1, 1, 1)
    bound = 2.0 ** -20 * (a.sqrt() * x0.to(F64).abs() + (1 - a).sqrt() * nz.to(F64).abs())
    assert bool(((noisy - R.add_noise_ref(x0, nz, t, ac)).abs() <= bound).all()), "add_noise"
    loss, dpred = ops.mse_fwd_bwd(pred.cuda(), tgt.cuda())
    lref, dref = R.mse_ref(pred, tgt)
    assert abs(float(loss) / float(lref) - 1) <= 1e-5, (float(loss), float(lref))
    torch.testing.assert_close(dpred.cpu().to(F64), dref, rtol=2.0 ** -21, atol=0)
    loss, dpred = ops.mse_minsnr_fwd_bwd(pred.cuda(), tgt.cuda(), t.cuda(), ac.cuda(), 5.0)
    lref, dref = R.mse_minsnr_ref(pred, tgt, t, ac, 5.0)
    assert abs(float(loss) / float(lref) - 1) <= 1e-5, (float(loss), float(lref))
    torch.testing.assert_close(dpred.cpu().to(F64), dref, rtol=2.0 ** -19, atol=0)


# ------------------------------------------------------------------------------------------------ CLIP / splice helpers
@pytest.mark.parametrize("res,kpad", [(224, 592), (336, 640)])
def test_clip_patchify_and_assemble_bitexact(res, kpad):
    ops = _ops()
    N, p, C = 2, 14, 1024
    img = torch.randn(N, 3, res, res, generator=_g(res)).to(BF)
    cols = ops.clip_patchify(img.cuda(), p, kpad).cpu()
    assert kpad > 3 * p * p and torch.equal(cols, R.clip_patchify_ref(img, p, kpad))
    P = (res // p) ** 2
    patches = torch.randn(N * P, C, generator=_g(res + 1)).to(BF)
    cls = torch.randn(C, generator=_g(res + 2)).to(BF)
    pos = torch.randn(P + 1, C, generator=_g(res + 3)).to(BF)
    out = ops.clip_assemble(patches.cuda(), cls.cuda(), pos.cuda(), N, P).cpu()
    want = torch.cat([cls.expand(N, 1, C), patches.view(N, P, C)], dim=1) + pos          # bf16 + bf16: fp32 add, one rounding
    assert torch.equal(out, want)


def test_row_copies_segment_sums_and_zero_rows():
    ops = _ops()
    H = 1032                                                                 # 129 vectors per row
    g = _g(80)
    src = torch.randn(50, H, generator=g).to(BF)
    dst = torch.randn(40, H, generator=g).to(BF)
    dst_idx = torch.randperm(40, generator=g)[:20].to(torch.int32)
    src_idx = torch.randint(0, 5, (20,), generator=g, dtype=torch.int32)     # duplicate source rows
    got = ops.copy_rows_(dst.cuda(), dst_idx.cuda(), src.cuda(), src_idx.cuda()).cpu()
    want = dst.clone()
    want[dst_idx.long()] = src[src_idx.long()]
    assert torch.equal(got, want)
    got = ops.copy_rows_(dst.cuda(), dst_idx.cuda(), src.cuda(), src_idx.cuda(), accumulate=True).cpu()
    want = dst.clone()
    want[dst_idx.long()] = (dst[dst_idx.long()].float() + src[src_idx.long()].float()).to(BF)
    assert torch.equal(got, want)
    # segments: empty ones, a long one, repeated rows
    lens = torch.tensor([3, 0, 300, 1, 0, 17])
    seg = torch.cat([torch.zeros(1, dtype=torch.long), lens.cumsum(0)]).to(torch.int32)
    rows = torch.randint(0, 50, (int(lens.sum()),), generator=g, dtype=torch.int32)
    out = ops.segment_sum_rows(src.cuda(), seg.cuda(), rows.cuda(), lens.numel()).cpu()
    ref = R.segment_sum_rows_ref(src, seg, rows)
    abs_sum = R.segment_sum_rows_ref(src.abs(), seg, rows)
    _close_bf16(out, ref, atol=2.0 ** -20 * abs_sum, what="segment_sum_rows")
    assert torch.equal(out[1], torch.zeros(H, dtype=BF)) and torch.equal(out[4], torch.zeros(H, dtype=BF))
    idx = torch.tensor([3, 17, 5], dtype=torch.int32)
    got = ops.zero_rows_(dst.cuda(), idx.cuda()).cpu()
    want = dst.clone()
    want[idx.long()] = 0
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ wrapper input checks
def _bad_inputs():
    d = "cuda"
    x = torch.zeros(2, 4, 6, 16, device=d, dtype=BF)
    nc = x.transpose(1, 2)                                                   # [2, 6, 4, 16], not contiguous
    w4 = torch.zeros(4, 16, 3, 3, device=d, dtype=BF)
    sched = torch.zeros(5, device=d, dtype=torch.int32)
    step = torch.zeros(1, device=d, dtype=torch.int32)
    h = torch.zeros(1, 8, 4, 6, device=d)
    wq, bq = torch.zeros(8, 8, device=d, dtype=BF), torch.zeros(8, device=d, dtype=BF)
    z = torch.zeros(1, 4, 4, 6, device=d)
    ops = _ops()
    return {
        "geglu_bwd dtype": lambda: ops.geglu_bwd(torch.zeros(4, 8, device=d), torch.zeros(4, 16, device=d, dtype=BF)),
        "geglu_bwd layout": lambda: ops.geglu_bwd(torch.zeros(8, 4, device=d, dtype=BF).t(), torch.zeros(4, 16, device=d, dtype=BF)),
        "upsample2x layout": lambda: ops.upsample2x(nc),
        "upsample2x dtype": lambda: ops.upsample2x(x.float()),
        "upsample2x_bwd layout": lambda: ops.upsample2x_bwd(nc),
        "upsample2x_bwd dtype": lambda: ops.upsample2x_bwd(x.float()),
        "im2col_s2 layout": lambda: ops.im2col_s2(nc),
        "im2col_s2 dtype": lambda: ops.im2col_s2(x.float(), pad=0),
        "col2im_s2 dtype": lambda: ops.col2im_s2(torch.zeros(12, 144, device=d), 2, 4, 6, 16),
        "col2im_s2 layout": lambda: ops.col2im_s2(torch.zeros(144, 12, device=d, dtype=BF).t(), 2, 4, 6, 16),
        "conv_out_bwd dtype": lambda: ops.conv_out_bwd(torch.zeros(2, 4, 4, 6, device=d, dtype=BF), w4, 16),
        "conv_out_bwd layout": lambda: ops.conv_out_bwd(torch.zeros(2, 4, 6, 4, device=d).transpose(2, 3), w4, 16),
        "timestep_embedding dtype": lambda: ops.timestep_embedding(sched.long(), step, 2, 320),
        "timestep_embedding step dtype": lambda: ops.timestep_embedding(sched, step.long(), 2, 320),
        "timestep_embedding_batch dtype": lambda: ops.timestep_embedding_batch(sched.long(), 320),
        "timestep_embedding_batch layout": lambda: ops.timestep_embedding_batch(sched[::2], 320),
        "vae_sample layout": lambda: ops.vae_sample(torch.zeros(1, 8, 6, 4, device=d).transpose(2, 3), wq, bq, z, 0.18),
        "vae_sample dtype": lambda: ops.vae_sample(h, wq.float(), bq, z, 0.18),
        "vae_sample z dtype": lambda: ops.vae_sample(h, wq, bq, z.to(BF), 0.18),
    }


def test_wrappers_reject_bad_inputs_before_launch():
    ops = _ops()
    torch.cuda.synchronize()
    for name, call in _bad_inputs().items():
        n0 = ops.LAUNCHES.count
        with pytest.raises(AssertionError):
            call()
        assert ops.LAUNCHES.count == n0, f"{name}: launched before rejecting"
    # groupnorm_bwd now checks weight and bias for the device too
    x = torch.zeros(1, 4, 4, 64, device="cuda", dtype=BF)
    st = torch.zeros(1, 32, 2, device="cuda")
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        ops.groupnorm_bwd(x, x, torch.ones(64, dtype=BF), torch.zeros(64, dtype=BF), st, 32, True)
    torch.cuda.synchronize()


def test_column_copies_reject_misaligned_rows():
    """copy_cols / copy_cols2 move 16-byte vectors: a base pointer that is not 16-byte aligned is refused by the library."""
    ops = _ops()
    buf = torch.zeros(1 + 4 * 16, device="cuda", dtype=BF)
    src = buf[1:].view(4, 16)                                                # contiguous, 2-byte aligned
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        ops.copy_cols_(src, torch.zeros(4, 32, device="cuda", dtype=BF), 8)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        ops.split_channels(buf[1:].view(1, 2, 2, 16), 8)
    torch.cuda.synchronize()

"""Host-side checks of the 3x3 convolution's float64 references and comparison (oracle/conv3x3_oracle.py), no GPU:

* the references agree with independent formulations (unfold + matmul, autograd through F.conv2d, the adjoint identity), and
  `ops.conv3x3_dgrad_weight` run as a forward conv is conv2d_input;
* the comparison tests/test_conv3x3_gpu.py applies rejects a kernel that is subtly wrong: faults a kernel could plausibly have (a
  dropped tap, a misplaced 128-column seam, a row that wraps into the next, an image that leaks into its tile neighbour, the wrong
  image's time embedding) are injected into the reference on the GPU test's own inputs, and C_ACC stays 10x below the smallest of
  their signals;
* the split-K planner (host code) still sends the GPU test's cases down the paths the test asserts;
* the image-size rule the pipelines apply.
"""
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import conv3x3_oracle as R

BF = torch.bfloat16
F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _lib():
    from dreamllm_b200 import _lib
    _lib.build()
    return _lib.lib()


def _unfold_conv(x_nhwc, w_k):
    """Explicit im2col in the kernel's K order (r, s, c) and one float64 matmul."""
    N, H, W, Cin = x_nhwc.shape
    cols = F.unfold(x_nhwc.to(F64).permute(0, 3, 1, 2), 3, padding=1)           # [N, Cin * 9, HW], (c, r, s)
    cols = cols.reshape(N, Cin, 9, H * W).permute(0, 3, 2, 1).reshape(N * H * W, 9 * Cin)
    return (cols @ w_k.to(F64).T).reshape(N, H, W, -1)


# ------------------------------------------------------------------------------------------------ references
@pytest.mark.parametrize("N,H,W,Cin,Cout", [(2, 5, 7, 3, 4), (1, 1, 6, 8, 8), (3, 4, 4, 64, 16)])
def test_forward_ref_matches_unfold_matmul(N, H, W, Cin, Cout):
    x = torch.randn(N, H, W, Cin, generator=_g(1)).to(BF)
    w_k = torch.randn(Cout, 9 * Cin, generator=_g(2)).to(BF)
    assert torch.allclose(R.conv3x3_acc(x, w_k), _unfold_conv(x, w_k), rtol=1e-12, atol=1e-12)


def test_epilogue_rounds_where_the_kernel_rounds():
    acc = torch.tensor([[[[1.0 + 2.0 ** -8, 3.0]]]], dtype=F64)                   # 1 + 2^-8 is a bf16 tie: rounds to even (1.0)
    bias = torch.tensor([0.0, 2.0 ** -8], dtype=BF)
    rowbias = torch.tensor([[2.0 ** -12, 0.0]], dtype=BF)
    residual = torch.tensor([[[[2.0 ** -9, -3.0]]]], dtype=BF)
    t, y, _ = R.epilogue_ref(acc, bias, rowbias, residual)
    assert t.flatten().tolist() == [1.0078125, 3.0]                             # 1 + 2^-9 + 2^-12 rounds up; 3 + 2^-8 rounds to 3
    assert y.flatten().tolist() == [1.0078125, 0.0]                             # + 2^-9 is under half an ulp
    assert R.epilogue_ref(acc)[1].flatten().tolist() == [1.0, 3.0]


@pytest.mark.parametrize("N,H,W,Cin,Cout", [(2, 5, 7, 4, 3), (1, 8, 8, 64, 8)])
def test_dgrad_ref_matches_autograd_and_adjoint(N, H, W, Cin, Cout):
    weight = torch.randn(Cout, Cin, 3, 3, generator=_g(3)).to(BF)
    dy = torch.randn(N, H, W, Cout, generator=_g(4)).to(BF)
    x = torch.randn(N, H, W, Cin, generator=_g(5), dtype=F64).requires_grad_(True)
    y = F.conv2d(x.permute(0, 3, 1, 2), weight.to(F64), padding=1).permute(0, 2, 3, 1)
    (y * dy.to(F64)).sum().backward()
    dx = R.conv3x3_dgrad_ref(dy, weight)
    assert torch.allclose(dx, x.grad, rtol=1e-12, atol=1e-12)
    w_k = weight.permute(0, 2, 3, 1).reshape(Cout, -1)
    lhs = (R.conv3x3_acc(x.detach(), w_k) * dy.to(F64)).sum()
    rhs = (x.detach() * dx).sum()
    assert abs(float(lhs - rhs)) <= 1e-10 * float((x.detach().abs() * R.conv3x3_dgrad_ref(dy.abs(), weight.abs())).sum())


def test_dgrad_weight_as_forward_conv_is_conv2d_input():
    from dreamllm_b200 import ops
    weight = torch.randn(16, 64, 3, 3, generator=_g(6)).to(BF)
    dy = torch.randn(2, 6, 8, 16, generator=_g(7)).to(BF)
    w_dg = ops.conv3x3_dgrad_weight(weight)
    assert w_dg.shape == (64, 9 * 16)
    assert torch.allclose(R.conv3x3_acc(dy, w_dg), R.conv3x3_dgrad_ref(dy, weight), rtol=1e-12, atol=1e-12)
    assert torch.equal(R._w4(ops.conv3x3_weight(weight)), weight.to(F64))


def test_term_mass_bounds_the_sum():
    x = torch.randn(1, 4, 8, 64, generator=_g(8)).to(BF)
    w_k = torch.randn(8, 9 * 64, generator=_g(9)).to(BF)
    assert bool((R.conv3x3_acc(x, w_k).abs() <= R.term_mass(x, w_k)).all())
    assert torch.allclose(R.term_mass(x, w_k), _unfold_conv(x.abs(), w_k.abs()), rtol=1e-12)


# ------------------------------------------------------------------------------------------------ injected faults
def _tap_conv(x_nhwc, w_k, src):
    """float64 conv written as nine gathers: output pixel m = (n, h, w) takes tap (r, s) from flat pixel src(r, s) (-1: padding)."""
    N, H, W, Cin = x_nhwc.shape
    xf = torch.cat([x_nhwc.to(F64).reshape(N * H * W, Cin), torch.zeros(1, Cin, dtype=F64)])
    wk = w_k.to(F64).reshape(w_k.shape[0], 9, Cin)
    out = 0
    for r in range(3):
        for s in range(3):
            idx = src(r, s)
            out = out + xf[torch.where(idx >= 0, idx, N * H * W)] @ wk[:, 3 * r + s].T
    return out.reshape(N, H, W, -1)


def _coords(N, H, W):
    n, h, w = torch.meshgrid(torch.arange(N), torch.arange(H), torch.arange(W), indexing="ij")
    return n.flatten(), h.flatten(), w.flatten()


def _src_true(N, H, W):
    n, h, w = _coords(N, H, W)

    def src(r, s):
        hh, ww = h + r - 1, w + s - 1
        ok = (hh >= 0) & (hh < H) & (ww >= 0) & (ww < W)
        return torch.where(ok, (n * H + hh) * W + ww, -1)
    return src


def _src_fault(kind, N, H, W):
    n, h, w = _coords(N, H, W)
    true = _src_true(N, H, W)

    def src(r, s):
        hh, ww = h + r - 1, w + s - 1
        if kind == "drop_tap":                       # one K block's tap never loaded
            return true(r, s) if (r, s) != (0, 0) else torch.full_like(n, -1)
        if kind == "seam_edge":                      # the tile's own box edge taken for the plane's: no tap crosses w = 128k
            return torch.where(ww // 128 == w // 128, true(r, s), -1)
        if kind == "seam_shift":                     # tiles past the first of a row fetched one column to the right
            ww = torch.where(w >= 128, ww + 1, ww)
            ok = (hh >= 0) & (hh < H) & (ww >= 0) & (ww < W)
            return torch.where(ok, (n * H + hh) * W + ww, -1)
        if kind == "row_wrap":                       # column padding lost: w = W-1 reads the next row's first pixel
            p = hh * W + ww
            return torch.where((p >= 0) & (p < H * W), n * H * W + p, -1)
        if kind == "image_leak":                     # row padding lost between images of a tile: h = -1 / H reads the neighbour
            m = (n * H + hh) * W + ww
            return torch.where((ww >= 0) & (ww < W) & (m >= 0) & (m < N * H * W), m, -1)
        raise ValueError(kind)
    return src


# (fault, case): each on the GPU test's own inputs, at the plane where the kernel could make it
FAULT_CASES = [("drop_tap", R.CASES[8]), ("seam_edge", R.CASES[0]), ("seam_shift", R.CASES[0]), ("row_wrap", R.CASES[6]),
               ("image_leak", R.CASES[12]), ("rowbias_wrong_image", R.CASES[12])]


def _fault_signal(kind, case):
    """(slack_needed of the faulted reference against the true one, faulted y, (t, y, mass) of the true reference)."""
    x, w_k, bias, rowbias, residual = R.conv_inputs(case)
    N, H, W = case.N, case.H, case.W
    acc = R.conv3x3_acc(x, w_k)
    mass = R.term_mass(x, w_k)
    t, y, pre = R.epilogue_ref(acc, bias, rowbias)
    if kind == "rowbias_wrong_image":                # the last pixel of every image takes the next image's time embedding
        rb = rowbias.to(F64)[:, None, None, :].expand(N, H, W, -1).clone()
        rb[:, H - 1, W - 1] = rowbias.to(F64).roll(-1, 0)
        y_f = R.bf16r(acc + bias.to(F64) + rb)
    else:
        acc_f = _tap_conv(x, w_k, _src_fault(kind, N, H, W))
        y_f = R.epilogue_ref(acc_f, bias, rowbias)[1]
    return R.slack_needed(y_f.to(BF), t, y, mass), y_f, (t, y, mass, pre)


def test_tap_formulation_is_the_reference():
    case = R.CASES[12]
    x, w_k = R.conv_inputs(case)[:2]
    assert torch.allclose(_tap_conv(x, w_k, _src_true(case.N, case.H, case.W)), R.conv3x3_acc(x, w_k), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("kind,case", FAULT_CASES, ids=[f[0] for f in FAULT_CASES])
def test_criterion_rejects_injected_fault(kind, case):
    signal, y_f, (t, y, mass, pre) = _fault_signal(kind, case)
    assert signal >= 10 * R.C_ACC, f"{kind}: fault signal {signal:.3g} is not 10x above C_ACC = {R.C_ACC:.3g}"
    with pytest.raises(AssertionError):
        R.check_conv(y_f.to(BF), t, y, mass, pre, what=kind)
    R.check_conv(y.to(BF), t, y, mass, pre, what="unfaulted")


# ------------------------------------------------------------------------------------------------ split-K plan of the GPU cases
def test_split_k_paths_of_the_gpu_cases_are_pinned():
    """ops.conv3x3 asks for a split-K workspace when N H W <= 4096; the planner (host code, 132 SMs) then splits or not.  Both paths
    must stay covered by the GPU test, which asserts the same flags on the device."""
    L = _lib()
    got = [c.N * c.H * c.W <= 4096 and L.dllm_conv3x3_splitk_workspace_bytes(c.N, c.H, c.W, c.Cin, c.Cout) > 0 for c in R.CASES]
    assert got == [c.split for c in R.CASES]
    assert {R.box_class(c.H, c.W) for c in R.CASES if c.split} == {"seam", "row", "rows", "images"}
    assert {R.box_class(c.H, c.W) for c in R.CASES if not c.split} == {"seam", "row", "rows", "images"}
    assert L.dllm_conv3x3_splitk_workspace_bytes(1, 0, 8, 64, 8) == 0


def test_gpu_cases_cover_every_box_class():
    classes = {}
    for c in R.CASES:
        classes.setdefault(R.box_class(c.H, c.W), []).append(c)
    assert set(classes) == {"seam", "row", "rows", "images"}
    for cls, cs in classes.items():
        assert any(c.H > c.W for c in cs) and any(c.H < c.W for c in cs), cls
    assert {c.W for c in R.CASES} == {512, 256, 128, 64, 32, 16, 8, 4}
    assert {c.Cin for c in R.CASES} == {64, 128, 320, 1280, 2560} and {c.Cout for c in R.CASES} == {8, 128, 320, 328, 1280}
    partial = [c for c in classes["images"] if (c.N * c.H * c.W) % 128]
    assert {(c.H, c.W, c.N) for c in partial} >= {(8, 8, 1), (8, 8, 3), (4, 4, 3)}
    for c in R.CASES:                                # host float64 reference <= ~2 GFLOP each
        assert 2 * c.N * c.H * c.W * 9 * c.Cin * c.Cout <= 2.0e9, c.id


# ------------------------------------------------------------------------------------------------ the image-size rule
def test_plane_rule_mirrors_the_box_plan():
    from dreamllm_b200 import ops
    for H in range(0, 70):
        for W in list(range(0, 40)) + [48, 64, 96, 128, 192, 256, 384, 512, 640]:
            assert ops.conv3x3_plane_ok(H, W) == (R.box_plan(H, W) is not None), (H, W)


def _head(unet_cfg):
    from dreamllm_b200.unet import SD21, SDXL
    from dreamllm_b200.vae import SDVAE
    cfg = {"sd21": SD21, "sdxl": SDXL}[unet_cfg]
    return types.SimpleNamespace(resolution=512, unet=types.SimpleNamespace(cfg=cfg), vae_decoder=types.SimpleNamespace(cfg=SDVAE))


@pytest.mark.parametrize("unet_cfg", ["sd21", "sdxl"])
def test_pipeline_refuses_unsupported_sizes_up_front(unet_cfg):
    from dreamllm_b200 import ops
    from dreamllm_b200.modeling_plugins import StableDiffusionHead
    head = _head(unet_cfg)
    emb = torch.zeros(1, 4, 8)
    call = lambda h, w: StableDiffusionHead._pipeline_inputs(head, h, w, 1, None, emb, None, "latent")  # noqa: E731
    for h, w in ((512, 512), (1024, 1024), (128, 128), (512, 1024), (2048, 256), (64, 64)):
        assert call(h, w)[:2] == (h, w)
    for h, w in ((768, 768), (512, 768), (384, 512), (640, 640), (1024, 1152)):
        with pytest.raises(ValueError, match="not supported"):
            call(h, w)
    levels = len(head.unet.cfg["block_out_channels"])
    assert ops.diffusion_conv_planes(512, 768, levels, 4)[:2] == [(64, 96), (32, 48)]
    assert (768, 512) in ops.diffusion_conv_planes(768, 512, levels, 4)

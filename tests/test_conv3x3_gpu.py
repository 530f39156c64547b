"""The implicit-GEMM 3x3 convolution (`dllm_conv3x3_nhwc[_ws]`, `ops.conv3x3`) against float64 (oracle/conv3x3_oracle.py), element by
element, at every tile shape its 4-D TMA box takes: part of a row with a seam at w = 128k, one row, several rows, several whole images
(with a partial last tile); non-square planes; K blocks crossing the tap boundary (Cin / 64 = 1 .. 40); an N-tile tail (Cout 328).

Criterion (`check_conv`): |got - ref| <= one bf16 ulp per rounding point + C_ACC x term_mass (the fp32 accumulation's slack, scaled by
sum |x| |w| of that output), and at most 1 % of the elements differ from the reference at all, not counting those within that slack of
a rounding midpoint.  The structure probes compare bits.
"""
import pytest
import torch

from oracle import conv3x3_oracle as R

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
F64 = torch.float64
ERR_SHAPE = -1


def _ops():
    from dreamllm_b200 import ops
    return ops


def _L():
    from dreamllm_b200._lib import lib
    return lib()


def _p(t):
    return 0 if t is None else t.data_ptr()


def _direct(x, w_k, bias=None, rowbias=None, residual=None):
    """dllm_conv3x3_nhwc: never split."""
    N, H, W, Cin = x.shape
    Cout = w_k.shape[0]
    y = torch.empty(N, H, W, Cout, device=x.device, dtype=BF)
    rc = _L().dllm_conv3x3_nhwc(_p(x), _p(w_k), _p(y), N, H, W, Cin, Cout, _p(bias), _p(rowbias), _p(residual),
                                torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    return y


_REF = {}


def _reference(case):
    """(inputs, accumulator, term_mass) of a case, computed once per module run."""
    if case not in _REF:
        inp = R.conv_inputs(case)
        _REF[case] = (inp, R.conv3x3_acc(inp[0], inp[1]), R.term_mass(inp[0], inp[1]))
    return _REF[case]


def _uses_split(case):
    c = case
    return c.N * c.H * c.W <= 4096 and _L().dllm_conv3x3_splitk_workspace_bytes(c.N, c.H, c.W, c.Cin, c.Cout) > 0


# ------------------------------------------------------------------------------------------------ (a) float64 parity
@pytest.mark.parametrize("path", ["ops", "direct"])
@pytest.mark.parametrize("epi", R.EPILOGUES)
@pytest.mark.parametrize("case", R.CASES, ids=[c.id for c in R.CASES])
def test_conv3x3_vs_float64(case, epi, path):
    ops = _ops()
    (x, w_k, bias, rowbias, residual), acc, mass = _reference(case)
    b, rb, rs = R.epilogue_operands(epi, bias, rowbias, residual)
    t, y, pre = R.epilogue_ref(acc, b, rb, rs)
    dev = [v.cuda() if v is not None else None for v in (x, w_k, b, rb, rs)]
    if path == "ops":
        assert _uses_split(case) == case.split, "the split-K plan of this case changed"
        got = ops.conv3x3(*dev[:2], bias=dev[2], rowbias=dev[3], residual=dev[4])
    else:
        got = _direct(*dev)
    got = got.cpu()
    print(f"conv3x3 slack {R.box_class(case.H, case.W)} {case.id} {epi} {path}: {R.slack_needed(got, t, y, mass):.3e}")
    R.check_conv(got, t, y, mass, pre, what=f"{case.id} {epi} {path}")


# ------------------------------------------------------------------------------------------------ (b) exact structure probes
# (N, H, W, Cin, [(n, h, w, c), ...]): a single 1.0 at the first / last row and column of an image, on both sides of a 128-column
# seam, at the last column of a row that shares its tile with the next row, and at the last / first pixel of images sharing a tile.
PROBES = [
    (1, 3, 256, 128, [(0, 1, 127, 70), (0, 1, 128, 3), (0, 0, 0, 0), (0, 2, 255, 127)]),
    (2, 1, 512, 64, [(0, 0, 383, 5), (0, 0, 511, 63), (1, 0, 0, 9)]),
    (1, 4, 128, 64, [(0, 1, 127, 1), (0, 2, 0, 2), (0, 3, 127, 60)]),
    (2, 8, 32, 128, [(0, 0, 31, 64), (0, 3, 0, 1), (1, 7, 31, 127), (0, 7, 31, 0)]),
    (1, 16, 16, 64, [(0, 7, 15, 8), (0, 8, 0, 9)]),
    (5, 4, 8, 64, [(0, 3, 7, 1), (1, 0, 0, 2), (3, 3, 7, 3), (4, 0, 0, 4), (4, 3, 7, 5)]),
    (3, 4, 4, 128, [(0, 3, 3, 65), (1, 0, 0, 0), (2, 3, 3, 127)]),
    (3, 8, 8, 64, [(0, 7, 7, 3), (1, 0, 0, 4), (2, 7, 0, 5)]),
]


@pytest.mark.parametrize("N,H,W,Cin,pixels", PROBES, ids=[f"{R.box_class(p[1], p[2])}-{p[0]}x{p[1]}x{p[2]}" for p in PROBES])
def test_conv3x3_single_pixel_stencil_bitexact(N, H, W, Cin, pixels):
    """Each output is one product w * 1.0 or exactly zero: the result must be the 3x3 stencil of weights around the pixel, and zero in
    the next row, across the seam and in the neighbouring image of the same tile."""
    Cout = 136
    w_k = torch.randn(Cout, 9 * Cin, generator=torch.Generator().manual_seed(N * H * W + Cin)).to(BF)
    for n, h, w, c in pixels:
        x = torch.zeros(N, H, W, Cin, dtype=BF)
        x[n, h, w, c] = 1.0
        want = R.conv3x3_acc(x, w_k)
        got = _direct(x.cuda(), w_k.cuda()).cpu().to(F64)
        assert int((want != 0).any(-1).sum()) == sum(1 for dh in (-1, 0, 1) for dw in (-1, 0, 1) if 0 <= h + dh < H and 0 <= w + dw < W)
        if not torch.equal(got, want):
            bad = (got != want).any(-1).nonzero().tolist()
            raise AssertionError(f"1.0 at {(n, h, w, c)}: outputs wrong at pixels {bad[:8]} (of {len(bad)})")


@pytest.mark.parametrize("path", ["fused", "splitk"])
@pytest.mark.parametrize("N,H,W", [(5, 4, 8), (3, 8, 8), (3, 4, 4), (2, 8, 16), (2, 1, 256)])
def test_conv3x3_rowbias_per_image_bitexact(N, H, W, path):
    """x = 0: every pixel of image n is bf16(bias + rowbias[n]) (the fp32 sum of two bf16 values of like magnitude is exact), through
    the fused epilogue and through splitk_reduce_kernel; a tile holding several images switches rows of rowbias inside the tile."""
    ops = _ops()
    Cin, Cout = 320, 328
    g = torch.Generator().manual_seed(N * H * W)
    bias = (0.5 + torch.rand(Cout, generator=g)).to(BF)
    rowbias = (0.5 + torch.rand(N, Cout, generator=g)).to(BF)
    w_k = torch.randn(Cout, 9 * Cin, generator=g).to(BF)
    x = torch.zeros(N, H, W, Cin, dtype=BF, device="cuda")
    want = R.bf16r(bias.to(F64) + rowbias.to(F64))[:, None, None, :].expand(N, H, W, Cout)
    split = _uses_split(R.Case(N, H, W, Cin, Cout, True))
    if path == "splitk":
        assert split, "this plane no longer runs split-K"
        got = ops.conv3x3(x, w_k.cuda(), bias=bias.cuda(), rowbias=rowbias.cuda())
    else:
        got = _direct(x, w_k.cuda(), bias.cuda(), rowbias.cuda())
    assert torch.equal(got.cpu().to(F64), want)


# ------------------------------------------------------------------------------------------------ (c) dgrad
@pytest.mark.parametrize("N,H,W,Cin,Cout", R.DGRAD_CASES, ids=[f"{R.box_class(c[1], c[2])}-{c[0]}x{c[1]}x{c[2]}-{c[3]}" for c in R.DGRAD_CASES])
def test_conv3x3_dgrad_vs_float64(N, H, W, Cin, Cout):
    """dx = ops.conv3x3(dy, ops.conv3x3_dgrad_weight(w)) against conv2d_input, and <conv(x), g> = <x, conv^T(g)> on the kernel's
    outputs within the sum of their allowances."""
    ops = _ops()
    g = torch.Generator().manual_seed(Cin + H)
    weight = (torch.randn(Cout, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).to(BF)
    dy = torch.randn(N, H, W, Cout, generator=g).to(BF)
    x = torch.randn(N, H, W, Cin, generator=g).to(BF)
    wd = weight.cuda()
    w_dg = ops.conv3x3_dgrad_weight(wd)
    dx = ops.conv3x3(dy.cuda(), w_dg).cpu()
    dx_pre = R.conv3x3_dgrad_ref(dy, weight)
    dx_y = R.bf16r(dx_pre)
    dx_mass = R.term_mass(dy, w_dg.cpu())
    print(f"conv3x3 slack dgrad {N}x{H}x{W}-{Cin}: {R.slack_needed(dx, None, dx_y, dx_mass):.3e}")
    R.check_conv(dx, None, dx_y, dx_mass, dx_pre, what="dgrad")

    w_k = ops.conv3x3_weight(wd)
    y = ops.conv3x3(x.cuda(), w_k).cpu()
    y_pre = R.conv3x3_acc(x, w_k.cpu())
    y_ref = R.bf16r(y_pre)
    y_mass = R.term_mass(x, w_k.cpu())
    R.check_conv(y, None, y_ref, y_mass, y_pre, what="forward")
    lhs = float((y.to(F64) * dy.to(F64)).sum())
    rhs = float((x.to(F64) * dx.to(F64)).sum())
    bound = float((R.allowance(None, y_ref, y_mass) * dy.to(F64).abs()).sum() + (x.to(F64).abs() * R.allowance(None, dx_y, dx_mass)).sum())
    assert abs(lhs - rhs) <= bound, (lhs, rhs, bound)


# ------------------------------------------------------------------------------------------------ (d) refusals
# (H, W, Cin, Cout): planes no box describes (W not a multiple of 128 nor a divisor of it; H not a multiple of the rows per tile; a
# tile that cannot hold whole images), empty planes, channels off the K block / the 8-column store
REFUSED = [(8, 96, 64, 8), (8, 48, 64, 8), (8, 24, 64, 8), (8, 12, 64, 8), (2, 192, 64, 8), (6, 32, 64, 8), (12, 8, 64, 8),
           (0, 8, 64, 8), (8, 0, 64, 8), (8, 8, 96, 8), (8, 8, 32, 8), (8, 8, 64, 12), (8, 8, 64, 0)]


@pytest.mark.parametrize("H,W,Cin,Cout", REFUSED)
def test_conv3x3_refuses_before_launch(H, W, Cin, Cout):
    ops = _ops()
    N = 1
    x = torch.zeros(N, H, W, Cin, dtype=BF, device="cuda")
    w_k = torch.zeros(max(Cout, 1), 9 * Cin, dtype=BF, device="cuda")
    y = torch.zeros(N * max(H, 1) * max(W, 1) * max(Cout, 8) + 8, dtype=BF, device="cuda")
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    L = _L()
    assert L.dllm_conv3x3_nhwc(_p(x), _p(w_k), _p(y), N, H, W, Cin, Cout, 0, 0, 0, s) == ERR_SHAPE
    assert L.dllm_conv3x3_nhwc_ws(_p(x), _p(w_k), _p(y), N, H, W, Cin, Cout, 0, 0, 0, _p(ws), ws.numel(), s) == ERR_SHAPE
    if Cout > 0:
        with pytest.raises(RuntimeError, match=r"dllm_conv3x3_nhwc(_ws)? failed: invalid shape"):
            ops.conv3x3(x, w_k[:Cout])
    assert not bool(y.any()), "a refused call wrote to its output"


def test_conv3x3_misaligned_workspace_runs_unsplit():
    """A workspace that is not 16-byte aligned makes conv3x3_nhwc_ws fall back to the unsplit launch: bit-identical to
    dllm_conv3x3_nhwc."""
    case = R.Case(3, 8, 8, 320, 328, True)
    x, w_k, bias, rowbias, residual = (v.cuda() for v in R.conv_inputs(case))
    N, H, W, Cin, Cout = case.N, case.H, case.W, case.Cin, case.Cout
    wsb = _L().dllm_conv3x3_splitk_workspace_bytes(N, H, W, Cin, Cout)
    assert wsb > 0
    ws = torch.empty(wsb + 16, dtype=torch.uint8, device="cuda")
    y = torch.empty(N, H, W, Cout, dtype=BF, device="cuda")
    for b, rb, rs in ((None, None, None), (bias, rowbias, None), (bias, None, residual)):
        rc = _L().dllm_conv3x3_nhwc_ws(_p(x), _p(w_k), _p(y), N, H, W, Cin, Cout, _p(b), _p(rb), _p(rs), _p(ws) + 8, wsb,
                                       torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        assert torch.equal(y, _direct(x, w_k, b, rb, rs))


# ------------------------------------------------------------------------------------------------ the Python rule == the C rule
def test_plane_rule_matches_the_library():
    """ops.conv3x3_plane_ok (what the pipelines check image sizes with) against dllm_conv3x3_nhwc's return code on a sweep of planes,
    N = 1, Cin = 64, Cout = 8."""
    ops = _ops()
    Hs = list(range(1, 41)) + [64, 96, 128, 132]
    Ws = list(range(1, 21)) + [24, 32, 48, 64, 96, 128, 160, 192, 256, 384, 512]
    big = max(Hs) * max(Ws)
    x = torch.zeros(big * 64, dtype=BF, device="cuda")
    w_k = torch.zeros(8, 9 * 64, dtype=BF, device="cuda")
    y = torch.empty(big * 8, dtype=BF, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    L = _L()
    wrong = []
    accepted = 0
    for H in Hs:
        for W in Ws:
            rc = L.dllm_conv3x3_nhwc(_p(x), _p(w_k), _p(y), 1, H, W, 64, 8, 0, 0, 0, s)
            assert rc in (0, ERR_SHAPE), (H, W, rc)
            accepted += rc == 0
            if (rc == 0) != ops.conv3x3_plane_ok(H, W) or (rc == 0) != (R.box_plan(H, W) is not None):
                wrong.append((H, W, rc))
    torch.cuda.synchronize()
    assert not wrong, f"(H, W, rc) where the Python rule disagrees with the library: {wrong[:10]}"
    assert accepted > 100

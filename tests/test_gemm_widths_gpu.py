"""The intermediate N-tile widths (160 / 192 / 224, picked by the tile planner) in every mode they are instantiated for: forward NT with
the plain, bias + residual and activation epilogues, dgrad NN (192), and the implicit-GEMM conv at UNet widths.  Each is checked against
fp32 torch, and bit for bit against the same call with B zero-padded to a width the planner runs at 256: the N tile does not change the
K order in which an output element is summed."""
import pytest
import torch

pytestmark = pytest.mark.gpu

WIDTHS_KMAJOR = (160, 192, 224)


def _tile_n(M, N, K, b_mn):
    from dreamllm_b200._lib import lib
    return lib().dllm_gemm_tile_n(M, N, K, int(b_mn))


def _shape_for(width, b_mn, K):
    """Smallest (M, N) of a few M that the planner runs at `width`."""
    for M in (400, 4096, 16384):
        for N in range(64, 8192, 8):
            if _tile_n(M, N, K, b_mn) == width:
                return M, N
    raise AssertionError(f"no shape plans width {width} (b_mn={b_mn})")


def _padded_n(M, N, K, b_mn):
    """N' >= N (multiple of 64) that the planner runs unsplit at 256."""
    from dreamllm_b200._lib import lib
    for Np in range((N + 63) // 64 * 64, N + 4096, 64):
        if _tile_n(M, Np, K, b_mn) == 256 and lib().dllm_gemm_splitk_workspace_bytes(M, Np, K) == 0:
            return Np
    raise AssertionError(f"no padded width runs at 256 for {(M, N, K)}")


def _pad_rows(t, n):
    return torch.cat([t, torch.zeros((n - t.shape[0],) + tuple(t.shape[1:]), device=t.device, dtype=t.dtype)]).contiguous()


EPILOGUES = [  # (bias, residual, act)
    (False, False, 0),
    (True, False, 0),
    (True, True, 0),
    (True, False, 2),   # gelu
    (True, True, 3),    # silu, then the residual add
]


@pytest.mark.parametrize("bias,residual,act", EPILOGUES)
@pytest.mark.parametrize("width", WIDTHS_KMAJOR)
def test_fwd_width_epilogues(width, bias, residual, act):
    from dreamllm_b200 import ops
    K = 320
    M, N = _shape_for(width, False, K)
    g = torch.Generator(device="cuda").manual_seed(width + 7 * act)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    b = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16) if bias else None
    r = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16) if residual else None
    got = ops.gemm(a, w, bias=b, residual=r, act=act)

    ref = a.float() @ w.float().t()
    if bias or residual or act:
        y = ref + (b.float() if bias else 0)
        if act:
            y = y.to(torch.bfloat16).float()
            y = torch.nn.functional.gelu(y) if act == 2 else torch.nn.functional.silu(y)
        if residual:
            y = y.to(torch.bfloat16).float() + r.float()
        ref = y
    torch.testing.assert_close(got.float(), ref, rtol=2e-2, atol=3e-2)

    Np = _padded_n(M, N, K, False)
    rp = None
    if residual:
        rp = torch.zeros(M, Np, device="cuda", dtype=torch.bfloat16)
        rp[:, :N] = r
    wide = ops.gemm(a, _pad_rows(w, Np), bias=_pad_rows(b, Np) if bias else None, residual=rp, act=act)
    assert torch.equal(got, wide[:, :N])


def test_dgrad_width_192():
    from dreamllm_b200 import ops
    K = 640
    M, N = _shape_for(192, True, K)
    g = torch.Generator(device="cuda").manual_seed(11)
    dy = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(K, N, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    got = ops.gemm(dy, w, b_mn=True)
    torch.testing.assert_close(got.float(), dy.float() @ w.float(), rtol=2e-2, atol=3e-2)
    Np = _padded_n(M, N, K, True)
    wp = torch.zeros(K, Np, device="cuda", dtype=torch.bfloat16)
    wp[:, :N] = w
    assert torch.equal(got, ops.gemm(dy, wp, b_mn=True)[:, :N])


@pytest.mark.parametrize("epi", [False, True])
@pytest.mark.parametrize("side,cin,cout", [(64, 320, 320), (32, 640, 640)])
def test_conv_width(side, cin, cout, epi):
    """UNet 3x3 convs at the 64x64 (C 320) and 32x32 (C 640) levels of 4 samples: widths that fit C run unpadded."""
    from dreamllm_b200 import ops
    n = 4
    M, K = n * side * side, 9 * cin
    assert _tile_n(M, cout, K, False) in WIDTHS_KMAJOR
    g = torch.Generator(device="cuda").manual_seed(side + cout)
    x = torch.randn(n, side, side, cin, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(cout, K, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    bias = torch.randn(cout, device="cuda", generator=g).to(torch.bfloat16) if epi else None
    rowb = torch.randn(n, cout, device="cuda", generator=g).to(torch.bfloat16) if epi else None
    res = torch.randn(n, side, side, cout, device="cuda", generator=g).to(torch.bfloat16) if epi else None
    got = ops.conv3x3(x, w, bias=bias, rowbias=rowb, residual=res)

    w4 = w.float().view(cout, 3, 3, cin).permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w4, padding=1).permute(0, 2, 3, 1)
    if epi:
        ref = (ref + bias.float() + rowb.float()[:, None, None, :]).to(torch.bfloat16).float() + res.float()
    torch.testing.assert_close(got.float(), ref, rtol=2e-2, atol=3e-2)

    Np = _padded_n(M, cout, K, False)
    pad = Np - cout

    def padc(t):
        return None if t is None else torch.nn.functional.pad(t, (0, pad)).contiguous()
    wide = ops.conv3x3(x, _pad_rows(w, Np), bias=padc(bias), rowbias=padc(rowb), residual=padc(res))
    assert torch.equal(got, wide[..., :cout])

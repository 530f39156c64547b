"""wgmma GEMM parity (through the C ABI) vs an fp32 torch reference of the same contraction."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [
    # M, N, K
    (128, 256, 64),
    (256, 256, 128),
    (512, 4096, 4096),      # C1 q/k/v/o projection
    (384, 768, 320),        # tails in M, N; K not a multiple of 64
    (200, 264, 72),         # ragged everything (multiples of 8 only)
    (1024, 1408, 512),
    # widths served by the 128-wide N tile (pick_bn: less padded MMA work than 256): VAE C = 128, UNet C = 320 / 640
    (512, 128, 1152),
    (304, 320, 192),
    (1024, 640, 576),
]
MODES = [(False, False), (False, True), (True, True), (True, False)]


def _mk(M, N, K, a_mn, b_mn, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g).to(torch.bfloat16)
    b = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g).to(torch.bfloat16)
    A = a.float().t() if a_mn else a.float()
    Bm = b.float() if b_mn else b.float().t()
    return a, b, A @ Bm


@pytest.mark.parametrize("cta_pair", [0, 1])
@pytest.mark.parametrize("a_mn,b_mn", MODES)
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_fp32_out(M, N, K, a_mn, b_mn, cta_pair):
    from dreamllm_b200 import ops

    a, b, ref = _mk(M, N, K, a_mn, b_mn)
    c = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32, cta_pair=cta_pair)
    torch.cuda.synchronize()
    # bf16 inputs are exact in fp32; only the accumulation order differs
    torch.testing.assert_close(c, ref, rtol=1e-3, atol=1e-3 * (K ** 0.5))


@pytest.mark.parametrize("cta_pair", [0, 1])
def test_gemm_bf16_out_and_strided_views(cta_pair):
    from dreamllm_b200 import ops

    M, N, K = 640, 512, 256
    a, b, ref = _mk(M, N, K, False, False, seed=3)
    big = torch.zeros((M, 3 * N), device="cuda", dtype=torch.bfloat16)
    out = big[:, N:2 * N]                      # column-slice view: ldc = 3N
    ops.gemm(a, b, out=out, cta_pair=cta_pair)
    torch.cuda.synchronize()
    torch.testing.assert_close(out.float(), ref, rtol=1.6e-2, atol=1e-2 * (K ** 0.5))
    assert float(big[:, :N].abs().max()) == 0 and float(big[:, 2 * N:].abs().max()) == 0
    # A as a column-slice view (lda > K)
    abig = torch.randn((M, 2 * K), device="cuda").to(torch.bfloat16)
    c = ops.gemm(abig[:, K:], b, out_dtype=torch.float32, cta_pair=cta_pair)
    torch.testing.assert_close(c, abig[:, K:].float() @ b.float().t(), rtol=1e-3, atol=1e-3 * (K ** 0.5))


def test_gemm_linearity_full_size():
    """C2-sized projection (T=16384, 4096x4096): size-independent property instead of an oracle run."""
    from dreamllm_b200 import ops

    T, H = 16384, 4096
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn((T, H), device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn((H, H), device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    y = ops.gemm(x, w, out_dtype=torch.float32)
    y2 = ops.gemm((x * 2).to(torch.bfloat16), w, out_dtype=torch.float32)   # exact scaling in bf16
    torch.testing.assert_close(y2, 2 * y, rtol=0, atol=0)
    rows = torch.randint(0, T, (64,), device="cuda")
    torch.testing.assert_close(y[rows], x[rows].float() @ w.float().t(), rtol=1e-3, atol=2e-3)


@pytest.mark.parametrize("M,N,K,b_mn", [(256, 1280, 11520, False), (400, 4096, 4096, False), (400, 4096, 12288, True), (64, 320, 1280, False),
                                         (130, 264, 2048, True)])
def test_split_k_small_m_gemm(M, N, K, b_mn):
    """Small-M shapes run split-K (K slices on separate CTA pairs, fp32 partials in a workspace, epilogue in the reduce kernel): same
    result as the fp32 reference, and the fused-epilogue rounding points (bias in fp32, round, activation, round, residual, round)."""
    from dreamllm_b200 import ops
    from dreamllm_b200._lib import lib

    assert lib().dllm_gemm_splitk_workspace_bytes(M, N, K) > 0, "shape was expected to be split"
    g = torch.Generator(device="cuda").manual_seed(M + N)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    ref = a.float() @ (b.float() if b_mn else b.float().t())
    c = ops.gemm(a, b, b_mn=b_mn)
    torch.testing.assert_close(c.float(), ref, rtol=1.6e-2, atol=1e-2 * (K ** 0.5) * 0.05)
    if not b_mn:
        bias = (torch.randn(N, device="cuda", generator=g)).to(torch.bfloat16)
        res = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
        got = ops.linear(a, b, bias=bias, residual=res, act=ops.ACT_SILU)
        y = (ref + bias.float()).to(torch.bfloat16).float()
        y = torch.nn.functional.silu(y).to(torch.bfloat16).float()        # kernel rounds the activation output when a residual follows
        want = (y + res.float())
        torch.testing.assert_close(got.float(), want, rtol=2e-2, atol=3e-2)


def test_split_k_conv_small_plane_matches_unsplit(monkeypatch=None):
    """Implicit-GEMM conv on a small plane: split-K result == the unsplit kernel's up to fp32 summation order."""
    from dreamllm_b200 import ops
    from dreamllm_b200._lib import lib
    N, H, W, Ci, Co = 4, 8, 8, 640, 320
    assert lib().dllm_conv3x3_splitk_workspace_bytes(N, H, W, Ci, Co) > 0
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(N, H, W, Ci, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(Co, 9 * Ci, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    bias = torch.randn(Co, device="cuda", generator=g).to(torch.bfloat16)
    rowb = torch.randn(N, Co, device="cuda", generator=g).to(torch.bfloat16)
    res = torch.randn(N, H, W, Co, device="cuda", generator=g).to(torch.bfloat16)
    got = ops.conv3x3(x, w, bias=bias, rowbias=rowb, residual=res)
    # reference: torch conv2d in fp32 on the same bf16 values
    w4 = w.float().view(Co, 3, 3, Ci).permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w4, padding=1).permute(0, 2, 3, 1)
    ref = (ref + bias.float() + rowb.float()[:, None, None, :]).to(torch.bfloat16).float() + res.float()
    torch.testing.assert_close(got.float(), ref, rtol=2e-2, atol=3e-2)

"""The GEMM's two epilogues against each other.  A bf16 output view whose base is 16-byte aligned and whose row pitch is a multiple of 8
elements leaves through the staged epilogue (shared memory, TMA bulk tensor store clipped at the view's extents); any other bf16 view is
stored from registers.  Every case runs the same launch into both kinds of view and compares bits (the device erff / __expf cannot be
reproduced bit for bit in torch, so the direct store is the reference); cases without an activation are also compared with an
fp32-output launch followed by the epilogue's rounding sequence in torch.  The clipping cases pre-fill a larger buffer with a sentinel
and require every element outside the view to keep it."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
WIDTHS = (128, 160, 192, 224, 256)
SENTINEL = 1.0e30


def _L():
    from dreamllm_b200._lib import lib
    return lib()


def _tile_n(M, N, K, b_mn=False):
    return _L().dllm_gemm_tile_n(M, N, K, int(b_mn))


def _unsplit(M, N, K):
    return _L().dllm_gemm_splitk_workspace_bytes(M, N, K) == 0


def _shape_for(width, K, b_mn=False):
    """(M, N) with an M tail and N % 8 == 0 that the planner runs unsplit at `width`."""
    for M in (1000, 400, 4200):
        for N in range(8, 4096, 8):
            if _tile_n(M, N, K, b_mn) == width and _unsplit(M, N, K):
                return M, N
    raise AssertionError(f"no shape plans width {width} (b_mn={b_mn})")


def _odd_view(M, N, ld=None):
    """[M, N] bf16 view at row pitch `ld` whose base is one element past a 16-byte boundary: the direct-store epilogue."""
    ld = ld or N
    flat = torch.full((M * ld + 8,), SENTINEL, device="cuda", dtype=BF)
    v = flat[1:1 + M * ld].view(M, ld)[:, :N]
    assert v.data_ptr() % 16 == 2
    return v


def _rand(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(BF)


def _torch_epilogue(acc_f32, bias=None, rowbias_rows=None, residual=None):
    x = acc_f32
    if bias is not None:
        x = x + bias.float()
    if rowbias_rows is not None:
        x = x + rowbias_rows.float()
    if residual is not None:
        x = x.to(BF).float() + residual.float()
    return x.to(BF)


def _both(a, w, M, N, *, b_mn=False, bias=None, residual=None, act=0):
    from dreamllm_b200 import ops
    staged = ops.gemm(a, w, b_mn=b_mn, bias=bias, residual=residual, act=act)
    direct = ops.gemm(a, w, b_mn=b_mn, bias=bias, residual=residual, act=act, out=_odd_view(M, N))
    assert torch.equal(staged, direct)
    return staged


EPILOGUES = [  # (bias, residual, act)
    (False, False, 0), (True, False, 0), (False, True, 0), (True, True, 0),
    (True, False, 1), (True, False, 2), (True, False, 3), (True, True, 3),
]


@pytest.mark.parametrize("bias,residual,act", EPILOGUES)
@pytest.mark.parametrize("width", WIDTHS)
def test_forward_every_width(width, bias, residual, act):
    from dreamllm_b200 import ops
    K = 320
    M, N = _shape_for(width, K)
    g = torch.Generator(device="cuda").manual_seed(width + 13 * act + bias + 2 * residual)
    a, w = _rand(g, M, K), _rand(g, N, K, scale=0.05)
    b = _rand(g, N) if bias else None
    r = _rand(g, M, N + 24)[:, 8:8 + N] if residual else None          # ldr != N
    got = _both(a, w, M, N, bias=b, residual=r, act=act)
    if act == 0:
        acc = ops.gemm(a, w, out_dtype=torch.float32)
        assert torch.equal(got, _torch_epilogue(acc, b, None, r))


@pytest.mark.parametrize("K", [64, 320])
@pytest.mark.parametrize("N", [328, 8, 32008])
@pytest.mark.parametrize("M", [400, 1000, 1])
def test_tails(M, N, K):
    from dreamllm_b200 import ops
    assert _unsplit(M, N, K)
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a, w, b, r = _rand(g, M, K), _rand(g, N, K, scale=0.05), _rand(g, N), _rand(g, M, N)
    acc = ops.gemm(a, w, out_dtype=torch.float32)
    assert torch.equal(_both(a, w, M, N), acc.to(BF))
    assert torch.equal(_both(a, w, M, N, bias=b, residual=r), _torch_epilogue(acc, b, None, r))


@pytest.mark.parametrize("width", (128, 192, 256))
def test_dgrad(width):
    from dreamllm_b200 import ops
    K = 320
    M, N = _shape_for(width, K, b_mn=True)
    g = torch.Generator(device="cuda").manual_seed(width)
    dy, w = _rand(g, M, K), _rand(g, K, N, scale=0.05)
    got = _both(dy, w, M, N, b_mn=True)
    assert torch.equal(got, ops.gemm(dy, w, b_mn=True, out_dtype=torch.float32).to(BF))


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("M,inner", [(1000, 1280), (400, 64), (130, 192)])
def test_geglu(M, inner, bias):
    """inner = 64 and 192 leave the second half of the last 256-wide tile outside the output."""
    from dreamllm_b200 import ops
    K = 320
    g = torch.Generator(device="cuda").manual_seed(M + inner)
    x = _rand(g, M, K)
    wp, bp = ops.geglu_permute(_rand(g, 2 * inner, K, scale=0.05), _rand(g, 2 * inner) if bias else None)
    staged = ops.linear_geglu(x, wp, bp)
    direct = _odd_view(M, inner)
    rc = _L().dllm_gemm_bf16_geglu(x.data_ptr(), wp.data_ptr(), bp.data_ptr() if bias else 0, direct.data_ptr(), M, 2 * inner, K,
                                   x.stride(0), wp.stride(0), direct.stride(0), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    assert torch.equal(staged, direct)


@pytest.mark.parametrize("side,cin,cout", [(64, 320, 320), (32, 640, 640), (64, 64, 328)])
def test_conv3x3_bias_rowbias_residual(side, cin, cout):
    from dreamllm_b200 import ops
    n = 4 if side == 64 and cout == 320 else 5
    M = n * side * side
    assert M > 4096                                                       # never split-K
    g = torch.Generator(device="cuda").manual_seed(side + cout)
    x, w = _rand(g, n, side, side, cin), _rand(g, cout, 9 * cin, scale=0.02)
    bias, rowb, res = _rand(g, cout), _rand(g, n, cout), _rand(g, n, side, side, cout)
    staged = ops.conv3x3(x, w, bias=bias, rowbias=rowb, residual=res)
    direct = _odd_view(M, cout)
    rc = _L().dllm_conv3x3_nhwc(x.data_ptr(), w.data_ptr(), direct.data_ptr(), n, side, side, cin, cout, bias.data_ptr(),
                                rowb.data_ptr(), res.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    assert torch.equal(staged.view(M, cout), direct)
    plain = ops.conv3x3(x, w).view(M, cout)                               # plain-store instantiation of the conv
    direct.fill_(0)
    rc = _L().dllm_conv3x3_nhwc(x.data_ptr(), w.data_ptr(), direct.data_ptr(), n, side, side, cin, cout, 0, 0, 0,
                                torch.cuda.current_stream().cuda_stream)
    assert rc == 0 and torch.equal(plain, direct)


@pytest.mark.parametrize("epi", [False, True])
@pytest.mark.parametrize("M,N", [(1000, 328), (400, 8), (130, 1000)])
def test_views_are_clipped(M, N, epi):
    """The output as a column slice of a wider buffer and as a row block of a taller one: tiles overhang the view on both sides, and
    only the tensor map's extents keep the overhang out of the neighbours."""
    from dreamllm_b200 import ops
    K = 320
    g = torch.Generator(device="cuda").manual_seed(M * N + epi)
    a, w = _rand(g, M, K), _rand(g, N, K, scale=0.05)
    b, r = (_rand(g, N), _rand(g, M, N)) if epi else (None, None)
    want = ops.gemm(a, w, bias=b, residual=r, out=_odd_view(M, N))

    wide = torch.full((M + 3, N + 2 * 264), SENTINEL, device="cuda", dtype=BF)
    view = wide[:M, 264:264 + N]                                          # column slice; three sentinel rows below it
    assert view.data_ptr() % 16 == 0 and view.stride(0) % 8 == 0
    ops.gemm(a, w, bias=b, residual=r, out=view)
    assert torch.equal(view, want)
    mask = torch.ones_like(wide, dtype=torch.bool)
    mask[:M, 264:264 + N] = False
    assert bool((wide[mask] == SENTINEL).all())

    tall = torch.full((M + 2 * 136, N), SENTINEL, device="cuda", dtype=BF)
    if (136 * N) % 8 == 0:
        view = tall[136:136 + M]                                          # row block
        assert view.data_ptr() % 16 == 0
        ops.gemm(a, w, bias=b, residual=r, out=view)
        assert torch.equal(view, want)
        assert bool((tall[:136] == SENTINEL).all()) and bool((tall[136 + M:] == SENTINEL).all())


@pytest.mark.parametrize("pitch_pad,col0", [(5, 0), (8, 4), (3, 1)])
def test_views_no_tensor_map_can_describe(pitch_pad, col0):
    """Row pitch not a multiple of 8 elements, or a base off the 16-byte grid: the direct store, same bits, nothing else touched."""
    from dreamllm_b200 import ops
    M, N, K = 1000, 328, 320
    g = torch.Generator(device="cuda").manual_seed(pitch_pad)
    a, w, b, r = _rand(g, M, K), _rand(g, N, K, scale=0.05), _rand(g, N), _rand(g, M, N)
    want = ops.gemm(a, w, bias=b, residual=r)                             # staged
    buf = torch.full((M, N + 8 + pitch_pad), SENTINEL, device="cuda", dtype=BF)
    view = buf[:, col0:col0 + N]
    assert view.data_ptr() % 16 != 0 or view.stride(0) % 8 != 0
    ops.gemm(a, w, bias=b, residual=r, out=view)
    assert torch.equal(view, want)
    assert bool((buf[:, :col0] == SENTINEL).all()) and bool((buf[:, col0 + N:] == SENTINEL).all())

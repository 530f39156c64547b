"""The GEMM tile planner is host code: `dllm_gemm_tile_n` answers without a device (132 SMs assumed, an H100 SXM).  It picks the N-tile
width of the headline step's unsplit launches, and leaves every split-K shape, its width and its workspace as they were."""


def _lib():
    from dreamllm_b200 import _lib
    _lib.build()
    return _lib.lib()


# (M, N, K, b_mn) -> width: the stage-1 step's launches (UNet on 4 samples, 7B LLM on 400 tokens)
C5_WIDTHS = {
    (16384, 320, 320, 0): 160,       # UNet 64x64 level: linears, convs and their dgrads at C = 320
    (16384, 320, 2880, 0): 160,
    (4096, 640, 640, 0): 160,        # 32x32 level, C = 640
    (4096, 640, 5760, 0): 160,
    (16384, 960, 320, 0): 256,       # fused q|k|v of the 64x64 level: 4 waves of 256 tie 6 of 160
    (400, 12288, 4096, 0): 192,      # LLM q|k|v
    (400, 22016, 4096, 0): 224,      # LLM gate|up
    (400, 11008, 4096, 1): 192,      # LLM down_proj dgrad (NN)
    (512, 128, 1152, 0): 128,        # one 128-wide tile
    (8192, 12288, 4096, 0): 256,     # 7B training step (8192 tokens): many waves at any width
    (8192, 4096, 11008, 0): 256,
    (8192, 11008, 4096, 1): 256,
}


def test_c5_shapes_get_their_fitted_width():
    L = _lib()
    got = {s: L.dllm_gemm_tile_n(*s) for s in C5_WIDTHS}
    assert got == C5_WIDTHS


def test_mn_major_b_widths_are_multiples_of_64():
    """dgrad NN fetches B in 64-column boxes: only 128 / 192 / 256 exist for it."""
    L = _lib()
    seen = {L.dllm_gemm_tile_n(M, N, 4096, 1) for M in (400, 4096, 16384) for N in range(64, 8192, 8)}
    assert seen <= {128, 192, 256} and 192 in seen


def _split_plan_before(M, N, K, sms=132):
    """Split-K plan of the parent build (128 | 256 wide tiles): (width, slices, workspace bytes)."""
    bn = 128 if N <= 128 else 256
    mt, nt = (M + 127) // 128, (N + bn - 1) // bn
    tiles, num_kb = mt * nt, (K + 63) // 64
    ks = 1
    if tiles * 2 <= sms and num_kb >= 8:
        ks = min(sms // tiles, num_kb // 4, 16)
        if ks < 2:
            ks = 1
        if ks > 1:
            per = (num_kb + ks - 1) // ks
            ks = (num_kb + per - 1) // per
    return bn, ks, (ks * mt * 128 * N * 4 if ks > 1 else 0)


def test_split_k_shapes_are_unchanged():
    L = _lib()
    split = 0
    for M in (64, 128, 256, 400, 512, 1024, 4096):
        for N in (128, 320, 640, 1280, 4096, 11008):
            for K in (320, 1152, 2880, 4096, 5760, 11008, 11520, 22016):
                bn, ks, ws = _split_plan_before(M, N, K)
                assert L.dllm_gemm_splitk_workspace_bytes(M, N, K) == ws, (M, N, K)
                if ks > 1:
                    split += 1
                    for b_mn in (0, 1):
                        assert L.dllm_gemm_tile_n(M, N, K, b_mn) == bn, (M, N, K, b_mn)
    assert split > 20

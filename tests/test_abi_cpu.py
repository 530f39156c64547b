"""CPU-side checks of the C-ABI boundary: the library builds for sm_90a, loads without a GPU, exports every
symbol include/dreamllm_sm100.h declares, and the product path fails loudly (no CPU fallback)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "dreamllm_sm100.h")).read()
    return sorted(set(re.findall(r"\b(dllm_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from dreamllm_b200 import _lib
    _lib.build()
    L = _lib.lib()
    syms = _declared_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/dreamllm_sm100.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature"
    assert L.dllm_version() >= 100
    assert L.dllm_error_string(-1).decode().startswith("invalid")
    # pure host queries work without a device
    assert L.dllm_attn_bwd_workspace_bytes(2, 100, 4, 128) == 2 * 128 * 4 * 2 * 4


def test_sass_contains_wgmma_and_tma():
    """The shipped cubin is Hopper-native: warpgroup MMA (HGMMA) fed by TMA loads (UTMALDG), every kernel built for sm_90a."""
    import subprocess
    from dreamllm_b200 import _lib
    _lib.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for mnem in ("HGMMA", "UTMALDG"):
        assert mnem in sass, mnem
    assert "HMMA.16816" not in sass      # no legacy mma.sync path
    archs = set(re.findall(r"arch = (sm_\w+)", sass))
    assert archs == {"sm_90a"}, archs


def test_tile_gemm_mma_instructions_are_issued_back_to_back():
    """Regression guard for the issue path of the warpgroup MMAs.  Inside one wgmma commit group (the HGMMAs up to the one that carries
    `gsb0`) no WARPGROUP.DEPBAR, barrier or call may separate two HGMMAs: a function call reachable from the wgmma region (printf in the
    bounded mbarrier wait) once made ptxas serialise every wgmma (C7510, a DEPBAR after each HGMMA).  And the HGMMAs of a group follow
    each other closely (median gap <= 8 instructions): rebuilding the smem descriptors per K step put 11-13 instructions between them."""
    import statistics
    import subprocess
    from dreamllm_b200 import _lib
    _lib.build()
    bdir = os.path.join(os.path.dirname(_lib.LIB_PATH), "build")
    checked = 0
    for obj in ("gemm_sm90.o", "attn_sm90.o"):
        sass = subprocess.run(["cuobjdump", "-sass", os.path.join(bdir, obj)], capture_output=True, text=True).stdout
        for body in re.split(r"Function : ", sass)[1:]:
            name = body.split("\n", 1)[0]
            ins = [ln for ln in body.splitlines() if re.match(r"\s+/\*[0-9a-f]{4}\*/", ln)]
            pos = [i for i, ln in enumerate(ins) if "HGMMA" in ln]
            if len(pos) < 4:
                continue
            gaps = []
            for a, b in zip(pos, pos[1:]):
                if "gsb0" in ins[a]:                       # end of a commit group: waits may follow
                    continue
                assert not any(m in ln for ln in ins[a + 1:b] for m in ("DEPBAR", "BAR.SYNC", "CALL")), (name[:80], ins[a + 1:b])
                gaps.append(b - a)
            assert gaps and statistics.median(gaps) <= 8, (name[:80], gaps)
            checked += 1
    assert checked >= 30, checked


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    from dreamllm_b200 import ops
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMDecoderLayer
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.gemm(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))
    layer = DreamLLMDecoderLayer(DreamLLMConfig(hidden_size=256, intermediate_size=512, num_attention_heads=2)).to(torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        layer(torch.zeros(1, 8, 256, dtype=torch.bfloat16))


def test_product_does_not_import_oracle():
    """oracle/ is test infrastructure: nothing under dreamllm_b200/ may reference it."""
    for dp, _, files in os.walk(os.path.join(ROOT, "dreamllm_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, os.path.join(dp, f)


def test_host_only_entry_points_answer_without_a_gpu():
    """Version, error strings and the `*_workspace_bytes` queries are pure host code: callable on the build box (no compute is launched)."""
    from dreamllm_b200 import _lib
    L = _lib.lib()
    assert L.dllm_version() >= 100
    msgs = {code: L.dllm_error_string(code).decode() for code in (0, -1, -2, -3, -4, -5, -6)}
    assert len(set(msgs.values())) == len(msgs) and all(msgs.values())
    assert L.dllm_rmsnorm_bwd_workspace_bytes(16384, 4096) >= 64 * 4096 * 4 > 0          # 64-way column partials (DESIGN §4)
    assert L.dllm_attn_bwd_workspace_bytes(8, 2048, 32, 128) >= 8 * 32 * 2048 * 4        # at least the fp32 row term D = rowsum(dO * O)
    assert L.dllm_attn_bwd_workspace_bytes(8, 2048, 32, 128) > L.dllm_attn_bwd_workspace_bytes(1, 512, 32, 128)
    assert L.dllm_groupnorm_workspace_bytes(16, 64 * 64, 32) > 0
    assert L.dllm_sumsq_workspace_bytes() == 132 * 4 * 4
    assert L.dllm_get_reserved_sms() == 0


def test_split_k_plan_never_has_an_empty_slice():
    """`dllm_gemm_splitk_workspace_bytes` / `dllm_conv3x3_splitk_workspace_bytes` are host code (132 SMs assumed without a device): the
    slice count they imply must divide the K blocks without an empty last slice.  The kernel gives every slice ceil(num_kb / ks) blocks, so
    ks = 16 over 90 blocks made slice 15 start past the end and store an accumulator no MMA had initialised (round 2, caught by the conv
    parity test on the GPU); small outputs must be split, full waves must not."""
    from dreamllm_b200 import _lib
    L = _lib.lib()

    def check(ws, M, N, K):
        mp = (M + 127) // 128 * 128
        assert ws % (mp * N * 4) == 0, (M, N, K, ws)
        ks = ws // (mp * N * 4)
        num_kb = (K + 63) // 64
        per = (num_kb + ks - 1) // ks
        assert ks >= 2 and (num_kb + per - 1) // per == ks and per >= 4, (M, N, K, ks, num_kb)
        return ks

    split = 0
    for M in (64, 128, 256, 400, 512, 1024, 4096):
        for N in (320, 640, 1280, 4096, 11008):
            for K in (320, 1152, 2880, 4096, 5760, 11520, 22016):
                ws = L.dllm_gemm_splitk_workspace_bytes(M, N, K)
                if ws:
                    check(ws, M, N, K)
                    split += 1
    assert split > 20
    assert L.dllm_gemm_splitk_workspace_bytes(16384, 4096, 4096) == 0                     # 1024 tiles: nothing to gain
    assert check(L.dllm_conv3x3_splitk_workspace_bytes(4, 8, 8, 640, 320), 256, 320, 9 * 640) == 15   # the shape that exposed the bug (90 K blocks)
    assert L.dllm_conv3x3_splitk_workspace_bytes(32, 64, 64, 320, 320) == 0


def test_optimizer_kernels_use_128_bit_accesses():
    """The HBM-bound optimizer-shard kernels stream through 128-bit vector loads / stores (LDG.E.128 / STG.E.128), no 32-bit bulk traffic."""
    import subprocess
    from dreamllm_b200 import _lib
    _lib.build()
    sass = subprocess.run(["cuobjdump", "-sass", "-fun", "adamw_kernel", _lib.LIB_PATH], capture_output=True, text=True).stdout
    if "adamw_kernel" not in sass:                       # older cuobjdump: -fun needs the mangled name; fall back to the whole dump
        sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"Function : ", sass)
    seen = 0
    for f in funcs:
        name = f.split("\n", 1)[0]
        if "adamw_kernel" in name or "sumsq_partial_kernel" in name:
            seen += 1
            wide = len(re.findall(r"LDG\.E\.128", f))
            narrow = len(re.findall(r"LDG\.E(?:\.CONSTANT)?\s", f))          # 32-bit loads: only the scalar sum-of-squares read is allowed
            assert wide >= (1 if "sumsq" in name else 4), (name, wide)
            assert narrow <= 1, (name, narrow)
            if "adamw" in name:
                assert len(re.findall(r"STG\.E\.128", f)) >= 3 and not re.findall(r"STG\.E\s", f), name
    assert seen >= 3


def test_hbm_kernels_issue_128_bit_memory_instructions():
    """north_star: "coalesced 128B vectorised HBM loads".  Round 1 shipped a `bfloat162[4]` vector struct that nvcc split into four
    32-bit LDG / STG per copy (VERDICT r1 item 9); the uint4-backed struct is now the only layout.  SASS of the shipped objects: every
    norm / rope / swiglu / groupnorm / geglu kernel moves its bf16 vectors with LDG.E.128 / STG.E.128, and no 32-bit *vector-path*
    access remains (scalar fp32 side arrays — rstd, stats — may still be 32-bit)."""
    import subprocess
    from dreamllm_b200 import _lib
    _lib.build()
    bdir = os.path.join(os.path.dirname(_lib.__file__), "build")

    def bodies(obj):
        sass = subprocess.run(["cuobjdump", "-sass", os.path.join(bdir, obj)], capture_output=True, text=True).stdout
        return {f.split("\n", 1)[0]: f for f in re.split(r"Function : ", sass)[1:]}
    checked = 0
    for obj, kernels in (("elementwise.o", ("rmsnorm_fwd_kernel", "rope_kernelILi128", "swiglu_fwd_kernel", "swiglu_bwd_kernel",
                                            "rmsnorm_bwd_dx_kernel", "layernorm_fwd")),
                         ("unet_ops.o", ("gn_partial_kernelILb0", "gn_apply_kernelILb0", "gn_apply_kernelILb1", "geglu_kernel",
                                         "geglu_bwd_kernel", "layernorm_bwd_warp_kernel"))):
        fs = bodies(obj)
        for k in kernels:
            hits = [b for n, b in fs.items() if k in n]
            assert hits, (obj, k, list(fs)[:5])
            for body in hits:
                wide = len(re.findall(r"(?:LDG|STG)\.E\.128", body))
                narrow16 = len(re.findall(r"(?:LDG|STG)\.E\.U16", body))
                assert wide >= 2 and narrow16 == 0, (k, wide, narrow16)
                checked += 1
    assert checked >= 12

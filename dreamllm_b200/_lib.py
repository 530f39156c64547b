"""ctypes loader (and in-tree builder) for libdreamllm_sm100.so — the C-ABI boundary (include/dreamllm_sm100.h).

There is NO fallback: if the shared library is missing or a call returns non-zero, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.environ.get("DLLM_LIB_PATH") or os.path.join(_HERE, "libdreamllm_sm100.so")   # env override: A/B builds in dev scripts
SOURCES = ["capi.cu", "gemm_sm90.cu", "elementwise.cu", "attn_sm90.cu", "unet_ops.cu", "optim.cu", "sdxl_ops.cu", "decode_sm90.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--use_fast_math", "-Xcompiler", "-fPIC", "-Xcompiler", "-O3",
]


def _needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(_CSRC, f) for f in os.listdir(_CSRC)] + [os.path.join(_HERE, "..", "include", "dreamllm_sm100.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    """nvcc-compile every .cu for sm_90a into dreamllm_b200/libdreamllm_sm100.so (in-tree, next to this module)."""
    if not force and not _needs_build():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    # A/B builds (with DLLM_LIB_PATH pointing at a second .so): e.g. DLLM_NVCC_EXTRA="-DDLLM_VEC128 -DDLLM_GN_GROUP2" (DESIGN.md §8)
    extra = os.environ.get("DLLM_NVCC_EXTRA", "").split()
    objs = []
    procs = []
    objdir = os.path.join(_HERE, "build") if LIB_PATH == os.path.join(_HERE, "libdreamllm_sm100.so") else LIB_PATH + ".objs"
    os.makedirs(objdir, exist_ok=True)          # A/B builds keep their objects next to their own .so
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, *extra, "-c", os.path.join(_CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{out}")
        if verbose and out:
            print(out)
    cmd = [nvcc, "-shared", "-o", LIB_PATH, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if out.returncode != 0:
        raise RuntimeError(f"link failed:\n{out.stdout}")
    return LIB_PATH


_vp, _i, _l, _f, _sz, _d = ctypes.c_void_p, ctypes.c_int, ctypes.c_long, ctypes.c_float, ctypes.c_size_t, ctypes.c_double

# name -> (restype, argtypes); mirrors include/dreamllm_sm100.h one-to-one
SIGNATURES = {
    "dllm_version": (_i, []),
    "dllm_error_string": (ctypes.c_char_p, [_i]),
    "dllm_set_reserved_sms": (_i, [_i]),
    "dllm_get_reserved_sms": (_i, []),
    "dllm_gemm_bf16": (_i, [_vp, _vp, _vp, _i, _i, _i, _l, _l, _l, _i, _i, _i, _i, _vp]),
    "dllm_rmsnorm_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _f, _vp]),
    "dllm_rmsnorm_bwd_workspace_bytes": (_sz, [_i, _i]),
    "dllm_rmsnorm_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _sz, _i, _i, _vp]),
    "dllm_rope_inplace": (_i, [_vp, _vp, _vp, _vp, _l, _i, _i, _i, _i, _vp]),
    "dllm_swiglu_fwd": (_i, [_vp, _vp, _l, _i, _i, _vp]),
    "dllm_swiglu_bwd": (_i, [_vp, _vp, _vp, _l, _i, _i, _vp]),
    "dllm_add_bf16": (_i, [_vp, _vp, _vp, _l, _vp]),
    "dllm_cross_entropy": (_i, [_vp, _vp, _vp, _f, _vp, _l, _i, _i, _i, _vp]),
    "dllm_embedding_fwd": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "dllm_embedding_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "dllm_attn_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _l, _l, _i, _f, _vp]),
    "dllm_attn_bwd_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "dllm_attn_bwd": (_i, [_vp] * 11 + [_sz, _i, _i, _i, _i, _l, _l, _l, _i, _f, _vp]),
    "dllm_gemm_bf16_ex": (_i, [_vp, _vp, _vp, _i, _i, _i, _l, _l, _l, _i, _i, _i, _i, _vp, _vp, _l, _i, _vp]),
    "dllm_layernorm_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _f, _vp]),
    "dllm_clip_patchify": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "dllm_clip_assemble": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "dllm_copy_rows": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "dllm_segment_sum_rows": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp]),
    "dllm_zero_rows": (_i, [_vp, _vp, _i, _i, _vp]),
    "dllm_attn_fwd_ex": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _l, _l, _l, _i, _f, _vp]),
    "dllm_attn_fwd_cache": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _l, _l, _l, _i, _f, _vp]),
    "dllm_attn_fwd_cache_mask": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _l, _l, _l, _i, _f, _vp]),
    "dllm_attn_fwd_gqa": (_i, [_vp] * 7 + [_i, _i, _i, _i, _i, _i, _i, _i, _l, _l, _l, _i, _f, _vp]),
    "dllm_attn_bwd_gqa": (_i, [_vp] * 11 + [_sz, _i, _i, _i, _i, _i, _i, _l, _l, _l, _l, _l, _i, _f, _vp]),
    "dllm_attn_probs_gqa": (_i, [_vp] * 6 + [_i] * 8 + [_l, _l, _i, _f, _vp]),
    "dllm_attn_fwd_varlen": (_i, [_vp] * 6 + [_i] * 6 + [_l, _l, _l, _i, _f, _vp]),
    "dllm_attn_bwd_varlen_workspace_bytes": (_sz, [_i, _i, _i]),
    "dllm_attn_bwd_varlen": (_i, [_vp] * 11 + [_sz] + [_i] * 6 + [_l, _l, _l, _l, _l, _i, _f, _vp]),
    "dllm_conv3x3_nhwc": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "dllm_groupnorm_workspace_bytes": (_sz, [_i, _i, _i]),
    "dllm_groupnorm_nhwc": (_i, [_vp, _vp, _vp, _vp, _vp, _sz, _i, _i, _i, _i, _f, _i, _vp]),
    "dllm_geglu": (_i, [_vp, _vp, _i, _i, _vp]),
    "dllm_upsample2x_nhwc": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "dllm_im2col_s2_nhwc": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "dllm_copy_cols": (_i, [_vp, _vp, _l, _i, _i, _i, _vp]),
    "dllm_conv_in": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "dllm_conv_out": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "dllm_gemm_splitk_workspace_bytes": (_sz, [_i, _i, _i]),
    "dllm_gemm_tile_n": (_i, [_i, _i, _i, _i]),
    "dllm_gemm_bf16_ws": (_i, [_vp, _vp, _vp, _i, _i, _i, _l, _l, _l, _i, _vp, _vp, _l, _i, _vp, _sz, _vp]),
    "dllm_conv3x3_splitk_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "dllm_conv3x3_nhwc_ws": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "dllm_gemm_bf16_geglu": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _l, _l, _l, _vp]),
    "dllm_im2col_in": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "dllm_nhwc_to_nchw_f32": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "dllm_timestep_embedding": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "dllm_timestep_embedding_batch": (_i, [_vp, _vp, _i, _i, _vp]),
    "dllm_sampler_step": (_i, [_vp, _vp, _vp, _vp, _vp, _f, _i, _i, _l, _vp]),
    "dllm_attn_bwd_ex": (_i, [_vp] * 11 + [_sz, _i, _i, _i, _i, _i, _l, _l, _l, _l, _l, _i, _f, _vp]),
    "dllm_groupnorm_stats": (_i, [_vp, _vp, _vp, _sz, _i, _i, _i, _i, _f, _vp]),
    "dllm_groupnorm_apply": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "dllm_groupnorm_bwd_nhwc": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _i, _i, _i, _i, _i, _vp]),
    "dllm_layernorm_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _f, _vp]),
    "dllm_layernorm_bwd_affine_workspace_bytes": (_sz, [_i, _i]),
    "dllm_layernorm_bwd_affine": (_i, [_vp] * 8 + [_sz, _i, _i, _f, _vp]),
    "dllm_quick_gelu": (_i, [_vp, _vp, _l, _vp]),
    "dllm_quick_gelu_bwd": (_i, [_vp, _vp, _vp, _l, _vp]),
    "dllm_geglu_bwd": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "dllm_upsample2x_bwd_nhwc": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "dllm_col2im_s2_nhwc": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "dllm_copy_cols2": (_i, [_vp, _vp, _l, _i, _i, _i, _i, _i, _vp]),
    "dllm_conv_out_bwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "dllm_add_noise": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _l, _vp]),
    "dllm_mse_fwd_bwd": (_i, [_vp, _vp, _vp, _vp, _l, _vp]),
    "dllm_mse_minsnr_fwd_bwd": (_i, [_vp, _vp, _vp, _vp, _f, _vp, _vp, _i, _l, _vp]),
    "dllm_softmax_rows": (_i, [_vp, _l, _i, _f, _vp]),
    "dllm_vae_sample": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _l, _f, _vp]),
    "dllm_adamw_step": (_i, [_vp, _vp, _vp, _vp, _vp, _l, _i, _d, _d, _d, _d, _d, _i, _vp, _d, _vp]),
    "dllm_sumsq_workspace_bytes": (_sz, []),
    "dllm_sumsq_bf16": (_i, [_vp, _l, _vp, _i, _vp, _sz, _vp]),
    "dllm_channel_sum_workspace_bytes": (_sz, [_i, _i, _i]),
    "dllm_channel_sum_nhwc": (_i, [_vp, _vp, _l, _i, _f, _i, _i, _i, _vp, _sz, _vp]),
    "dllm_time_ids_embedding": (_i, [_vp, _vp, _l, _i, _i, _i, _vp]),
    "dllm_silu_bf16": (_i, [_vp, _vp, _l, _vp]),
    "dllm_silu_bwd_bf16": (_i, [_vp, _vp, _vp, _l, _vp]),
    "dllm_broadcast_rows": (_i, [_vp, _vp, _i, _i, _i, _f, _vp]),
    "dllm_attn_decode_plan": (_i, [_i, _i, _i, _i, _vp, _vp]),
    "dllm_attn_decode_workspace_bytes": (_sz, [_i, _i, _i, _i, _i, _i]),
    "dllm_attn_decode": (_i, [_vp, _l, _vp, _vp, _vp, _vp, _i, _vp, _l, _vp, _sz, _i, _i, _i, _i, _i, _f, _i, _vp]),
    "dllm_rope_append_kv": (_i, [_vp, _l, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
}

_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing — run `python -c 'import __graft_entry__ as g; g.build()'`. "
                "dreamllm_b200 has no CPU / eager fallback by design."
            )
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the ABI is incomplete
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().dllm_error_string(rc).decode()
        raise RuntimeError(f"{what} failed: {msg} (code {rc})")

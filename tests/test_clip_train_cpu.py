"""Host side of the trainable CLIP tower: which parameters the plugin flags make trainable (against the reference's `requires_grad_`
calls applied to a transformers CLIPVisionModel), `fsdp_ignored_modules`, the ABI of the new kernels and their refusals.  No GPU needed."""
import ctypes

import pytest
import torch

CFG = dict(hidden_size=64, intermediate_size=256, num_hidden_layers=8, num_attention_heads=1, image_size=28, patch_size=14)
ROWS = [(True, True), (False, True), (False, False), (True, False)]      # (freeze_clip_vision_model, freeze_embedding_layers)


def _reference_trainable(freeze_tower, freeze_emb, select_layer):
    """transformers CLIPVisionModel with the reference's flag logic (omni/models/dreamllm/modeling_plugins.py:248-257), restated."""
    from transformers import CLIPVisionConfig, CLIPVisionModel
    m = CLIPVisionModel(CLIPVisionConfig(**CFG))
    m.requires_grad_(not freeze_tower)
    if not freeze_tower:
        for i in range(select_layer + 1, 0):
            m.vision_model.encoder.layers[i].requires_grad_(False)
        m.vision_model.post_layernorm.requires_grad_(False)
    m.vision_model.embeddings.requires_grad_(not freeze_emb)
    return {n for n, p in m.named_parameters() if p.requires_grad}, {n for n, _ in m.named_parameters()}


def _plugin(freeze_tower, freeze_emb, select_layer, freeze_projector=False):
    from dreamllm_b200.modeling_plugins import CLIPVisionEmbedding
    return CLIPVisionEmbedding(dict(CFG), embed_hidden_size=32, select_layer=select_layer, freeze_clip_vision_model=freeze_tower,
                               freeze_embedding_layers=freeze_emb, freeze_projector=freeze_projector)


@pytest.mark.parametrize("select_layer", [-2, 5])
@pytest.mark.parametrize("freeze_tower,freeze_emb", ROWS)
def test_trainable_set_matches_reference(freeze_tower, freeze_emb, select_layer):
    want, names = _reference_trainable(freeze_tower, freeze_emb, select_layer)
    clip = _plugin(freeze_tower, freeze_emb, select_layer)
    ours = {n for n, p in clip.clip_vision_model.named_parameters() if p.requires_grad}
    assert {n for n, _ in clip.clip_vision_model.named_parameters()} == names
    assert ours == want
    assert all(p.requires_grad for p in clip.projector.parameters())


@pytest.mark.parametrize("freeze_tower,freeze_emb", ROWS)
@pytest.mark.parametrize("freeze_projector", [False, True])
def test_fsdp_ignored_modules(freeze_tower, freeze_emb, freeze_projector):
    clip = _plugin(freeze_tower, freeze_emb, -2, freeze_projector)
    want = ([clip.clip_vision_model] if freeze_tower else []) + ([clip.projector] if freeze_projector else [])
    got = clip.fsdp_ignored_modules()
    assert len(got) == len(want) and all(a is b for a, b in zip(got, want))


def test_additional_post_layernorm_still_refused():
    from dreamllm_b200.modeling_plugins import CLIPVisionEmbedding
    with pytest.raises(ValueError, match="use_additional_post_layernorm"):
        CLIPVisionEmbedding(dict(CFG), embed_hidden_size=32, use_additional_post_layernorm=True, freeze_clip_vision_model=False)


def test_abi_signatures_and_workspace():
    from dreamllm_b200 import _lib
    L = _lib.lib()
    sig = {"dllm_layernorm_bwd_affine_workspace_bytes": 2, "dllm_layernorm_bwd_affine": 13, "dllm_quick_gelu": 4,
           "dllm_quick_gelu_bwd": 5}
    for name, n in sig.items():
        fn = getattr(L, name)
        assert fn.argtypes == _lib.SIGNATURES[name][1] and fn.restype == _lib.SIGNATURES[name][0] and len(fn.argtypes) == n
    # per-row (mean, rstd) as float2, then 64 row-split partials of dgamma and dbeta in fp32
    for T, H in ((1, 256), (577, 1024), (16 * 577, 1536)):
        assert L.dllm_layernorm_bwd_affine_workspace_bytes(T, H) == T * 8 + 64 * 2 * H * 4
    assert L.dllm_layernorm_bwd_affine_workspace_bytes(0, 1024) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="made-up addresses are passed only where no kernel can run; "
                    "test_clip_train_gpu.py checks the same refusals on real allocations")
def test_refusals_before_launch():
    """Bad pointers and shapes are refused by the library before anything touches a device."""
    from dreamllm_b200 import _lib
    L = _lib.lib()
    A, M = 1 << 20, (1 << 20) + 2                       # an aligned and a misaligned (2-byte offset) address: never dereferenced
    assert L.dllm_quick_gelu(M, A, 64, None) == -2
    assert L.dllm_quick_gelu(A, M, 64, None) == -2
    assert L.dllm_quick_gelu_bwd(A, A, M, 64, None) == -2
    assert L.dllm_quick_gelu(A, A, 12, None) != 0                         # n % 8
    ws = L.dllm_layernorm_bwd_affine_workspace_bytes(577, 1024)
    args = [A] * 8
    for i in (0, 1, 2, 4, 7):                            # dy, x, w, dx, workspace
        bad = list(args)
        bad[i] = M
        assert L.dllm_layernorm_bwd_affine(*bad, ws, 577, 1024, 1e-5, None) == -2
    assert L.dllm_layernorm_bwd_affine(*args, ws - 4, 577, 1024, 1e-5, None) != 0          # workspace too small
    assert L.dllm_layernorm_bwd_affine(*args, ws, 577, 1028, 1e-5, None) != 0             # H % 8
    assert L.dllm_layernorm_bwd_affine(*args, 1 << 30, 4, 1544, 1e-5, None) != 0          # wider than the widest warp variant
    nul = list(args)
    nul[5] = None                                                                          # no dgamma
    assert L.dllm_layernorm_bwd_affine(*nul, ws, 577, 1024, 1e-5, None) != 0


def test_wrappers_refuse_wrong_dtypes():
    from dreamllm_b200 import ops
    with pytest.raises(TypeError):
        ops.quick_gelu(torch.zeros(64))
    with pytest.raises(TypeError):
        ops.quick_gelu_bwd(torch.zeros(64, dtype=torch.bfloat16), torch.zeros(64, dtype=torch.float16))
    x = torch.zeros(4, 64, dtype=torch.bfloat16)
    with pytest.raises(TypeError):
        ops.layernorm_bwd_affine(x.float(), x, torch.ones(64, dtype=torch.bfloat16), 1e-5)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.quick_gelu(torch.zeros(64, dtype=torch.bfloat16))                              # no CPU fallback


def test_tower_without_trainable_parameters_keeps_the_frozen_path(monkeypatch):
    """The plugin's default flags leave every tower parameter frozen, so `hidden_state` takes the no_grad path."""
    from dreamllm_b200.clip_vision import CLIPVisionModel
    clip = _plugin(True, True, -2)
    called = []
    monkeypatch.setattr(CLIPVisionModel, "_hidden_state_frozen", lambda self, x, s: called.append("frozen"))
    monkeypatch.setattr(CLIPVisionModel, "_hidden_state_train", lambda self, x, s: called.append("train"))
    clip.clip_vision_model.hidden_state(None, -2)
    _plugin(True, False, -2).clip_vision_model.hidden_state(None, -2)
    assert called == ["frozen", "train"]

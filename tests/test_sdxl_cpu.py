"""SDXL head, host side: the UNet-XL architecture (parameter count, keys, shapes) on the native module and the from-spec oracle, the
oracle's addition embedding against a float64 closed form, the collator's add_time_ids, the new C ABI entries and the host-side errors."""
import math

import pytest
import torch

from oracle import unet_oracle as UO
from oracle import unet_xl_oracle as XO

SDXL_PARAMS = 2_567_463_684
SD21_PARAMS = 865_910_724


def test_sdxl_param_count_keys_and_shapes():
    from dreamllm_b200.unet import SDXL, UNet2DConditionModel
    assert SDXL == XO.SDXL
    with torch.device("meta"):
        m = UNet2DConditionModel(SDXL)
        r = XO.UNet2DConditionModel(SDXL)
    assert sum(p.numel() for p in m.parameters()) == SDXL_PARAMS
    assert sum(p.numel() for p in r.parameters()) == SDXL_PARAMS
    ms, rs = m.state_dict(), r.state_dict()
    assert [(k, tuple(v.shape)) for k, v in ms.items()] == [(k, tuple(v.shape)) for k, v in rs.items()]
    shapes = {k: tuple(v.shape) for k, v in ms.items()}
    assert shapes["add_embedding.linear_1.weight"] == (1280, 2816)
    assert shapes["add_embedding.linear_2.weight"] == (1280, 1280)
    assert shapes["mid_block.attentions.0.transformer_blocks.9.attn2.to_k.weight"] == (1280, 2048)
    assert "mid_block.attentions.0.transformer_blocks.10.norm1.weight" not in shapes
    assert shapes["down_blocks.2.attentions.1.transformer_blocks.9.ff.net.0.proj.weight"] == (10240, 1280)
    assert shapes["down_blocks.1.attentions.0.transformer_blocks.1.attn1.to_q.weight"] == (640, 640)
    assert shapes["up_blocks.0.attentions.2.transformer_blocks.9.norm3.weight"] == (1280,)
    assert shapes["up_blocks.1.attentions.2.transformer_blocks.1.attn2.to_v.weight"] == (640, 2048)
    assert not any(k.startswith(("down_blocks.0.attentions", "up_blocks.2.attentions")) for k in shapes)
    assert "down_blocks.2.downsamplers.0.conv.weight" not in shapes and "up_blocks.2.upsamplers.0.conv.weight" not in shapes
    assert shapes["up_blocks.0.resnets.2.conv1.weight"] == (1280, 1920, 3, 3)
    assert sum(1 for _ in m.blocks()) == 70 and sum(1 for _ in m.resnets()) == 17


def test_sd21_unchanged_by_the_new_options():
    from dreamllm_b200.unet import UNet2DConditionModel
    with torch.device("meta"):
        m = UNet2DConditionModel()
        r = XO.UNet2DConditionModel()
        o = UO.UNet2DConditionModel()
    assert sum(p.numel() for p in m.parameters()) == SD21_PARAMS == sum(p.numel() for p in r.parameters())
    assert list(m.state_dict()) == list(r.state_dict()) == list(o.state_dict())
    assert m.add_embedding is None and sum(1 for _ in m.blocks()) == 16


def test_oracle_addition_embedding_matches_float64_closed_form():
    torch.manual_seed(0)
    cfg = dict(block_out_channels=(64, 128), attention_head_dim=(1, 2), cross_attention_dim=32, down_attn=(False, True),
               up_attn=(True, False), transformer_layers_per_block=(1, 2), addition_embed_type="text_time", addition_time_embed_dim=256,
               projection_class_embeddings_input_dim=48 + 6 * 256)
    m = XO.UNet2DConditionModel(cfg)
    B = 3
    text = torch.randn(B, 48)
    ids = torch.tensor([[1024., 1024., 0., 0., 1024., 1024.], [768., 1344., 16., 32., 1024., 1024.], [512., 512., 7., 3., 896., 1152.]])
    add = m.add_embeds(text, ids, torch.float32)
    got = m.add_embedding(add)
    # float64 closed form: Timesteps(256, flip_sin_to_cos=True, shift 0) per id, [cos | sin], id-major; then linear_2(silu(linear_1(.)))
    half = 128
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64) / half)
    arg = ids.double()[:, :, None] * f[None, None]
    te = torch.cat([torch.cos(arg), torch.sin(arg)], dim=-1).reshape(B, -1)
    x = torch.cat([text.double(), te], -1)
    assert float((add.double() - x).abs().max()) < 2e-3          # fp32 sinusoid at arguments up to ~1.3e3
    l1, l2 = m.add_embedding.linear_1, m.add_embedding.linear_2
    z = x @ l1.weight.double().t() + l1.bias.double()
    want = (z * torch.sigmoid(z)) @ l2.weight.double().t() + l2.bias.double()
    assert torch.allclose(got.double(), want, rtol=1e-4, atol=1e-4)


class _Tok:
    pad_token_id = 0


def _examples(with_ids, all_none=False):
    ex = []
    for i, n in enumerate((5, 9, 7)):
        ids = torch.arange(1, n + 1)
        e = dict(input_ids=ids, attention_mask=torch.ones(n, dtype=torch.long), labels=ids.clone(), images=None, images_dm=None)
        if with_ids:
            e["add_time_ids"] = None if i == 1 or all_none else torch.tensor([[1024 + i, 1024, i, 0, 1024, 1024]])
        ex.append(e)
    return ex


@pytest.mark.parametrize("pack", [False, True])
def test_collator_emits_add_time_ids(pack):
    from dreamllm_b200.collator import DataCollatorForDreamLLMDataset
    col = DataCollatorForDreamLLMDataset(_Tok(), pack=pack)
    out = col(_examples(True))
    assert out["add_time_ids"].shape == (2, 6)
    assert out["add_time_ids"][:, 0].tolist() == [1024, 1026]          # batch order, samples without ids skipped
    assert col(_examples(True, all_none=True))["add_time_ids"] is None
    base = col(_examples(False))
    assert "add_time_ids" not in base                                  # batches without the key are emitted as before
    for k, v in base.items():
        if isinstance(v, torch.Tensor):
            assert torch.equal(out[k], v), k


def test_new_abi_signatures():
    from dreamllm_b200 import _lib
    L = _lib.lib()
    want = {"dllm_channel_sum_workspace_bytes": 3, "dllm_channel_sum_nhwc": 11, "dllm_time_ids_embedding": 7, "dllm_silu_bf16": 4,
            "dllm_silu_bwd_bf16": 5, "dllm_broadcast_rows": 7}
    hdr = open(_lib.os.path.join(_lib._HERE, "..", "include", "dreamllm_sm100.h")).read()
    for name, nargs in want.items():
        assert name + "(" in hdr, name
        assert hasattr(L, name) and len(_lib.SIGNATURES[name][1]) == nargs, name
    # host-only query: one fp32 partial row per CTA chunk, none for an invalid shape
    ws = L.dllm_channel_sum_workspace_bytes(1, 16384, 320)
    assert ws > 0 and ws % (320 * 4) == 0
    assert L.dllm_channel_sum_workspace_bytes(2, 100, 12) == 0
    assert "sdxl_ops.cu" in _lib.SOURCES


def test_unet_config_errors():
    from dreamllm_b200.unet import SDXL, UNet2DConditionModel
    with torch.device("meta"):
        with pytest.raises(ValueError, match="addition_embed_type"):
            UNet2DConditionModel(dict(SDXL, addition_embed_type="text"))
        with pytest.raises(ValueError, match="transformer_layers_per_block"):
            UNet2DConditionModel(dict(SDXL, transformer_layers_per_block=(1, 2)))
        with pytest.raises(ValueError, match="head_dim must be 64"):
            UNet2DConditionModel(dict(SDXL, attention_head_dim=(5, 10, 10)))


def test_scheduler_config_is_checked(tmp_path):
    import json

    from dreamllm_b200.modeling_plugins import _check_scheduler_config
    p = tmp_path / "scheduler_config.json"
    p.write_text(json.dumps(dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                                 prediction_type="epsilon", steps_offset=1, timestep_spacing="leading", clip_sample=False)))
    _check_scheduler_config(str(p))
    p.write_text(json.dumps(dict(prediction_type="v_prediction", beta_start=0.00085)))
    with pytest.raises(ValueError, match="v_prediction"):
        _check_scheduler_config(str(p))


def test_causal_lm_add_time_ids_errors_before_any_kernel():
    """add_time_ids with a head that is not the XL head is refused on the host, before the decoder runs."""
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    m = DreamLLMForCausalMLM(DreamLLMConfig(vocab_size=64, hidden_size=64, intermediate_size=128, num_hidden_layers=1,
                                            num_attention_heads=1))
    with pytest.raises(ValueError, match="StableDiffusionXLHead"):
        m(input_ids=torch.ones(1, 4, dtype=torch.long), add_time_ids=torch.zeros(1, 6))

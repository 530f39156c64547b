"""Mint tests/golden/rescale_noise_cfg.npz and tests/golden/reference_config.json from the reference's own code.

    python -m oracle.gen_golden_surface /path/to/DreamLLM

Runs the reference's `_rescale_noise_cfg` (omni/models/dreamllm/modeling_plugins.py:658-669) and `DreamLLMConfig`
(omni/models/dreamllm/configuration_dreamllm.py:64-278) exec'd verbatim on CPU, and stores what they return, so that
tests/test_scheduler_cpu.py and tests/test_hf_surface_cpu.py compare against the reference without a checkout of it.
"""
from __future__ import annotations

import json
import os
import sys
import textwrap

import numpy as np
import torch

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def rescale_inputs():
    g = torch.Generator().manual_seed(0)
    text, uncond = torch.randn(3, 4, 8, 8, generator=g) * 1.3, torch.randn(3, 4, 8, 8, generator=g)
    return uncond + 7.5 * (text - uncond), text


def main(ref_root: str) -> None:
    src = open(os.path.join(ref_root, "omni/models/dreamllm/modeling_plugins.py")).read()
    a = src.index("    def _rescale_noise_cfg(")
    b = src.index("    @torch.no_grad()", a)
    ns = {"torch": torch}
    exec(textwrap.dedent(src[a:b]), ns)
    cfg, text = rescale_inputs()
    want = ns["_rescale_noise_cfg"](None, cfg, text, 0.7)
    np.savez(os.path.join(OUT, "rescale_noise_cfg.npz"), out=want.numpy())

    from transformers import PretrainedConfig

    class _Log:
        def warning(self, *a, **k):
            pass
        info = warning

    lines = open(os.path.join(ref_root, "omni/models/dreamllm/configuration_dreamllm.py")).read().split("\n")
    ns = dict(PretrainedConfig=PretrainedConfig, logger=_Log(), CLASS_KEY="_class_", NAME_KEY="_name_", PLUGIN_TYPE_KEY="_plugin_type_")
    exec("from __future__ import annotations\n" + "\n".join(lines[63:278]), ns)
    from dreamllm_b200.configuration_dreamllm import DreamLLMConfig
    ref = ns["DreamLLMConfig"]()
    keys = [k for k in DreamLLMConfig().to_dict() if k not in ("model_type", "rope_scaling")]
    defaults = json.loads(json.dumps({k: getattr(ref, k) for k in keys}, default=str))   # a copy: the update below mutates ref
    ref.update_special_tokens2ids_dict({"additional_special_tokens": ["<im_start>", "<dream_start>"], "bos_token": "<s>"}, _Tok())
    out = {"model_type": ref.model_type, "defaults": defaults, "special_tokens2ids_dict": ref.special_tokens2ids_dict}
    with open(os.path.join(OUT, "reference_config.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True, default=str)
        f.write("\n")


class _Tok:
    pad_token_id = 0

    def __len__(self):
        return 96

    def convert_tokens_to_ids(self, t):
        table = {"<im_start>": 90, "<im_patch>": 91, "<im_end>": 92, "<dream_start>": 93, "<dream_end>": 94, "<s>": 1, "</s>": 2}
        return [table[x] for x in t] if isinstance(t, list) else table[t]


if __name__ == "__main__":
    main(sys.argv[1])

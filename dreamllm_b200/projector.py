"""H100-native mirror of `omni/models/projector` (builder.py:10-22, mlp_projector.py:11-50, base_projector.py:8-36).

Same API: `build_projector(projector_cfg, in_hidden_size, out_hidden_size, bias)` returns a module with a `.projector`
submodule (state-dict key `projector.weight` / `projector.{0,2,..}.weight`), whose `forward(features | list)` returns a
**list** of tensors (callers take `[-1]`, modeling_plugins.py:325, :546).  Arithmetic: wgmma GEMM with fused bias /
GELU epilogue; backward = dgrad + wgrad GEMMs + bias column-sum.
"""
from __future__ import annotations

import os
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops

BF16 = torch.bfloat16


class _LinearFn(torch.autograd.Function):
    """y = act(x W^T + b).  act: 0 none, 2 gelu(erf).  Saves the pre-activation only when act != 0."""

    @staticmethod
    def forward(ctx, x, weight, bias, act):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        if act == 0:
            y = ops.linear(x2, weight, bias=bias)
            ctx.save_for_backward(x2, weight)
        else:
            pre = ops.linear(x2, weight, bias=bias)
            y = torch.nn.functional.gelu(pre) if act == ops.ACT_GELU else None  # backward needs `pre`; tiny tensors
            if y is None:
                raise ValueError("unsupported activation")
            ctx.save_for_backward(x2, weight, pre)
        ctx.act = act
        ctx.has_bias = bias is not None
        return y.view(*shp[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        if ctx.act == 0:
            x2, weight = ctx.saved_tensors
            dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        else:
            x2, weight, pre = ctx.saved_tensors
            dy2 = torch.ops.aten.gelu_backward(dy.reshape(-1, dy.shape[-1]).contiguous(), pre)
        dx = ops.linear_dgrad(dy2, weight) if ctx.needs_input_grad[0] else None
        dw = ops.linear_wgrad(dy2, x2) if ctx.needs_input_grad[1] else None
        db = None
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.float().sum(0).to(dy2.dtype)
        if dx is not None:
            dx = dx.view(*dy.shape[:-1], weight.shape[1])
        return dx, dw, db, None


def linear_fn(x, weight, bias=None, act=0):
    return _LinearFn.apply(x, weight, bias, act)


class BaseProjector(nn.Module):
    def load_model(self, model_name_or_path=None):
        if model_name_or_path is not None:
            for suffix, whole in ((".bin", True), (".pt", False)):
                f = os.path.join(model_name_or_path, f"{self.save_model_name}{suffix}") if os.path.isdir(model_name_or_path) else model_name_or_path
                if os.path.isfile(f) and f.endswith(suffix):
                    sd = torch.load(f, map_location="cpu", weights_only=True)
                    (self if whole else self.projector).load_state_dict(sd)
                    return True
        return False

    @property
    def save_model_name(self):
        return self.args.save_model_name + "_projector"

    @property
    def dtype(self):
        return next(self.projector.parameters()).dtype

    @property
    def device(self):
        return next(self.projector.parameters()).device


class LinearProjector(BaseProjector):
    def __init__(self, args, in_hidden_size, out_hidden_size, bias=True):
        super().__init__()
        self.args = args
        self.freeze_projector = args.freeze_projector
        self.depth = args.depth
        assert self.depth == 1, "LinearProjector now only supports depth=1"
        assert bias is not None, "bias should be set as True or False"
        self.projector = nn.Linear(in_hidden_size, out_hidden_size, bias=bias)

    def forward(self, features):
        if not isinstance(features, list):
            features = [features]
        with torch.set_grad_enabled(torch.is_grad_enabled() and not self.freeze_projector):
            return [linear_fn(f, self.projector.weight, self.projector.bias) for f in features]


class MLPProjector(BaseProjector):
    def __init__(self, args, in_hidden_size, out_hidden_size, bias=False):
        super().__init__()
        self.args = args
        self.freeze_projector = args.freeze_projector
        self.depth = args.depth
        assert self.depth > 1, "MLPProjector now only supports depth > 1, use linear if depth is 1"
        assert bias is not None, "bias should be set as True or False"
        modules = [nn.Linear(in_hidden_size, out_hidden_size, bias=bias)]
        for _ in range(1, self.depth):
            modules.append(nn.GELU())
            modules.append(nn.Linear(out_hidden_size, out_hidden_size, bias=bias))
        self.projector = nn.Sequential(*modules)

    def _run(self, f):
        lins = [m for m in self.projector if isinstance(m, nn.Linear)]
        for i, lin in enumerate(lins):
            f = linear_fn(f, lin.weight, lin.bias, act=ops.ACT_GELU if i + 1 < len(lins) else 0)
        return f

    def forward(self, features):
        if not isinstance(features, list):
            features = [features]
        with torch.set_grad_enabled(torch.is_grad_enabled() and not self.freeze_projector):
            return [self._run(f) for f in features]


def build_projector(projector_cfg, in_hidden_size, out_hidden_size, bias=None):
    cfg = SimpleNamespace(**projector_cfg)
    projector = getattr(cfg, "projector", None)
    if projector == "linear":
        return LinearProjector(args=cfg, in_hidden_size=in_hidden_size, out_hidden_size=out_hidden_size, bias=bias)
    if projector == "mlp":
        return MLPProjector(args=cfg, in_hidden_size=in_hidden_size, out_hidden_size=out_hidden_size, bias=bias)
    if projector in ("conv", "sam"):
        raise ValueError(f"projector '{projector}' is out of scope (unused by DreamLLM configs, SURVEY.md §2 row 4)")
    raise ValueError(f"Unknown projector: {projector} (supported: linear, mlp)")

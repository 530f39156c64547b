"""Data-parallel optimizer with sharded gradients + optimizer state (SURVEY.md §8f row 4).

What it replaces in the reference: stage-2 / SFT training runs HF Trainer with `fsdp="shard_grad_op auto_wrap"` wrapping every
`DreamLLMDecoderLayer` (projects/dreamllm/configs/stage2/base.py:91-94) and `optim="adamw_torch"` (:95; stage1/base.py:85),
gradient clipping at `max_grad_norm` (omni/train/trainer.py:800-807) and a cosine schedule with warm-up
(stage1/base.py:76-77).  `shard_grad_op` = parameters stay whole through forward and backward, gradients are reduce-scattered,
each rank owns 1/N of the optimizer state — ZeRO stage 2.

Design (one process per GPU, torch.distributed only as transport):

* parameters are re-seated as views of flat bf16 buckets (forward order inside a bucket, so the fused q|k|v and gate|up row blocks of
  `modeling_dreamllm._fuse_rows` stay adjacent); gradients land in a mirror-image flat bucket;
* as soon as the last gradient of a bucket is written (post-accumulate hooks, reverse order) the bucket is **reduce-scattered**
  asynchronously over NCCL (AVG), overlapping the rest of backward — half the bytes of DDP's all-reduce on the wire before the step;
* `step()`: local sum of squares of the owned gradient shards (`dllm_sumsq_bf16`) -> one 4-byte all-reduce -> per bucket one fused
  `dllm_adamw_step` launch over the owned shard (clip coefficient read from device memory: no host sync) -> asynchronous in-place
  **all-gather** of the updated bf16 parameter shard, one bucket behind the next bucket's AdamW kernel;
* optimizer state: fp32 master + fp32 exp_avg / exp_avg_sq for the owned 1/N only (default; 12 B/param/N), or `state_dtype=bf16`,
  which reproduces the arithmetic of the reference (torch.optim.AdamW stepping a model loaded in bf16: projects/dreamllm/train.py:68-70,
  :138) op for op.

The arithmetic is the CUDA kernel; `update_fn` / `sumsq_fn` exist so the CPU (gloo, world_size 2) tests can drive the host logic with
the checker's arithmetic — the product defaults raise on CPU tensors like every other op in this package.
"""
from __future__ import annotations

import math

import torch
import torch.distributed as dist

from .ddp import plan_runs

ALIGN = 128     # elements; every rank's shard starts 256-byte aligned and is a multiple of the kernels' 8-element vectors


def cosine_schedule_with_warmup(step: int, num_warmup_steps: int, num_training_steps: int, num_cycles: float = 0.5) -> float:
    """LR multiplier of `lr_scheduler_type="cosine"` + `warmup_ratio` (stage1/base.py:76-77) = transformers'
    `get_cosine_schedule_with_warmup` lambda."""
    if step < num_warmup_steps:
        return float(step) / float(max(1, num_warmup_steps))
    progress = float(step - num_warmup_steps) / float(max(1, num_training_steps - num_warmup_steps))
    return max(0.0, 0.5 * (1.0 + math.cos(math.pi * float(num_cycles) * 2.0 * progress)))


def decay_parameter_names(model) -> list:
    """Names of the parameters weight decay applies to — `Trainer.get_decay_parameter_names` (omni/train/trainer.py:381-390): everything
    that does not live inside a normalisation layer (`ALL_LAYERNORM_LAYERS` = nn.LayerNorm + DreamLLMRMSNorm, modeling_dreamllm.py:94) and has
    no "bias" in its name."""
    import torch.nn as nn

    from .modeling_dreamllm import DreamLLMRMSNorm
    norm_types = (nn.LayerNorm, DreamLLMRMSNorm)

    def walk(mod, prefix):
        names = []
        for cname, child in mod.named_children():
            if not isinstance(child, norm_types):
                names += walk(child, f"{prefix}{cname}.")
        names += [f"{prefix}{n}" for n in mod._parameters.keys()]      # parameters defined directly on this module
        return names

    return [n for n in walk(model, "") if "bias" not in n]


def optimizer_param_groups(model, weight_decay: float) -> list:
    """The two groups `Trainer.create_optimizer` builds (omni/train/trainer.py:436-446): trainable decay / no-decay parameters."""
    decay = set(decay_parameter_names(model))
    named = list(model.named_parameters())
    return [{"params": [p for n, p in named if n in decay and p.requires_grad], "weight_decay": weight_decay},
            {"params": [p for n, p in named if n not in decay and p.requires_grad], "weight_decay": 0.0}]


def training_step(model, optimizer, batch: dict, lr_scale: float = 1.0, accumulate: bool = False, grad_accum_steps: int = 1):
    """One data-parallel training step (`Trainer.training_step` + the optimizer part of `_inner_training_loop`,
    omni/train/trainer.py:1007-1049, :744-835): forward, backward (gradient buckets reduce-scatter as they fill), and — unless this is an
    accumulation micro-step — global-norm clip + sharded AdamW + parameter all-gather.
    With gradient accumulation every micro-step back-propagates `loss / grad_accum_steps` (accelerate's `backward` scales the loss by
    1 / gradient_accumulation_steps, and `training_step` returns `loss.detach() / gradient_accumulation_steps`, trainer.py:1043-1047), so
    the accumulated gradient — and with it `grad_norm` and the `max_grad_norm` clip — is the mean over micro-batches, as in the reference.
    Returns (scaled loss.detach(), grad_norm | None)."""
    model.train()
    ga = max(int(grad_accum_steps), 1)

    def fwd_bwd():
        out = model(**batch)
        loss = out.loss / ga if ga > 1 else out.loss
        loss.backward()
        return loss.detach()

    if accumulate:
        with optimizer.no_sync():
            return fwd_bwd(), None
    loss = fwd_bwd()
    norm = optimizer.step(lr_scale=lr_scale)
    optimizer.zero_grad()
    return loss, norm


def _cuda_update(g, p, m, v, master, **kw):
    from . import ops
    ops.adamw_step_(g, p, m, v, master, **kw)


def _cuda_sumsq(g, out):
    from . import ops
    ops.sumsq_bf16_(g, out, accumulate=True)


class _Bucket:
    __slots__ = ("params", "n", "padded", "chunk", "flat_param", "flat_grad", "pviews", "gviews", "gshard", "pshard", "master", "m", "v",
                 "pending", "seen", "ready", "launched", "work", "group", "gather")


class ShardedAdamW:
    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0,
                 max_grad_norm: float = 1.0, bucket_cap_mb: float = 256.0, process_group=None, state_dtype=torch.float32,
                 update_fn=None, sumsq_fn=None):
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if dist.is_initialized() else 0
        self.backend = dist.get_backend(process_group) if dist.is_initialized() else None
        self.defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay)
        self.max_grad_norm = float(max_grad_norm or 0.0)
        if state_dtype not in (torch.float32, torch.bfloat16):
            raise ValueError("state_dtype must be torch.float32 (sharded fp32 master) or torch.bfloat16 (reference arithmetic)")
        self.state_dtype = state_dtype
        self._update = update_fn or _cuda_update
        self._sumsq = sumsq_fn or _cuda_sumsq
        self.step_count = 0
        self.launched = 0            # reduce-scatters + all-gathers issued (tests / bench bookkeeping)
        self._attached = False
        self._sync = True            # False inside no_sync(): micro-batch gradients accumulate locally, nothing goes on the wire
        self._next = 0               # next bucket to reduce-scatter: collectives are issued in bucket order on every rank (ddp.py)
        params = list(params)
        if params and not isinstance(params[0], dict):
            params = [{"params": params}]
        self.param_groups = []
        self.buckets: list[_Bucket] = []
        cap = int(bucket_cap_mb * 1024 * 1024)
        seen = set()
        for g in params:
            grp = dict(self.defaults)
            grp.update({k: v for k, v in g.items() if k != "params"})
            plist = [p for p in g["params"] if p.requires_grad]
            for p in plist:
                if id(p) in seen:
                    raise ValueError("a parameter appears in more than one group")
                seen.add(id(p))
                if p.dtype != torch.bfloat16:
                    raise ValueError("ShardedAdamW steps bf16 parameters (cast the model with .to(torch.bfloat16))")
            grp["params"] = plist
            self.param_groups.append(grp)
            # buckets = consecutive runs of the group's parameters, cut by the gradient reducer's rule (q|k|v and gate|up stay adjacent)
            for run in plan_runs(plist, cap):
                self._make_bucket(run, grp)
        self._bucket_of = {}
        for b in self.buckets:
            for p in b.params:
                self._bucket_of[p] = b
        order = 0
        for g in self.param_groups:
            for p in g["params"]:
                p._zero_order = order            # registration (= forward) order, used to issue the parameter all-gathers front to back
                order += 1
        self._hooks = [p.register_post_accumulate_grad_hook(self._on_grad) for b in self.buckets for p in b.params]
        dev = self.buckets[0].flat_param.device if self.buckets else torch.device("cpu")
        self._ss = torch.zeros(1, dtype=torch.float32, device=dev)

    # ------------------------------------------------------------------------------------------ layout
    def _make_bucket(self, plist, group):
        b = _Bucket()
        b.params, b.group = plist, group
        b.n = sum(p.numel() for p in plist)
        unit = self.world * ALIGN
        b.padded = (b.n + unit - 1) // unit * unit
        b.chunk = b.padded // self.world
        dev = plist[0].device
        b.flat_param = torch.zeros(b.padded, dtype=torch.bfloat16, device=dev)
        b.flat_grad = torch.zeros(b.padded, dtype=torch.bfloat16, device=dev)
        b.pviews, b.gviews, off = {}, {}, 0
        with torch.no_grad():
            for p in plist:
                pv = b.flat_param[off:off + p.numel()].view(p.shape)
                pv.copy_(p.data)
                p.data = pv                                   # the parameter now lives in the bucket (identity / state-dict key unchanged)
                b.pviews[p] = pv
                b.gviews[p] = b.flat_grad[off:off + p.numel()].view(p.shape)
                p._dllm_grad_view = b.gviews[p]               # fused wgrad GEMMs write straight into the bucket (ddp.grad_out_view)
                off += p.numel()
        lo = self.rank * b.chunk
        b.pshard = b.flat_param[lo:lo + b.chunk]
        b.gshard = b.flat_grad[lo:lo + b.chunk] if self.world == 1 else torch.zeros(b.chunk, dtype=torch.bfloat16, device=dev)
        if self.state_dtype == torch.float32:
            b.master = b.pshard.float()
            b.m = torch.zeros(b.chunk, dtype=torch.float32, device=dev)
            b.v = torch.zeros(b.chunk, dtype=torch.float32, device=dev)
        else:
            b.master = None
            b.m = torch.zeros(b.chunk, dtype=torch.bfloat16, device=dev)
            b.v = torch.zeros(b.chunk, dtype=torch.bfloat16, device=dev)
        b.pending = set(plist)
        b.seen = set()               # parameters that received a gradient since zero_grad() (any micro-batch)
        b.ready = b.launched = False
        b.work = None
        b.gather = None
        self.buckets.append(b)

    def reseat(self):
        """Re-point parameters at their bucket views (after something replaced `p.data`, e.g. `module.to()`)."""
        with torch.no_grad():
            for b in self.buckets:
                for p in b.params:
                    v = b.pviews[p]
                    if p.data.data_ptr() != v.data_ptr():
                        v.copy_(p.data)
                        p.data = v

    # ------------------------------------------------------------------------------------------ backward side
    def _on_grad(self, p):
        b = self._bucket_of[p]
        v = b.gviews[p]
        if p.grad.data_ptr() != v.data_ptr():
            v.copy_(p.grad)
            p.grad = v
        b.seen.add(p)
        b.pending.discard(p)
        if not b.pending and self._sync and not b.launched:
            b.ready = True
            self._launch_ready()

    def _launch_ready(self):
        """In-order rule (torch DDP's): bucket i goes on the wire only after buckets 0..i-1 — every rank issues the same sequence of
        reduce-scatters even when its batch left some parameters without a gradient (those buckets are flushed by `step()`)."""
        while self._next < len(self.buckets) and self.buckets[self._next].ready:
            self._reduce_scatter(self.buckets[self._next])
            self._next += 1

    def _reduce_scatter(self, b):
        b.launched = True
        if self.world == 1:
            return
        if self.backend == "nccl":
            b.work = dist.reduce_scatter_tensor(b.gshard, b.flat_grad, op=dist.ReduceOp.AVG, group=self.pg, async_op=True)
        else:                                                 # gloo (CPU tests): no AVG op
            b.flat_grad.div_(self.world)
            b.work = dist.reduce_scatter_tensor(b.gshard, b.flat_grad, op=dist.ReduceOp.SUM, group=self.pg, async_op=True)
        self.launched += 1

    def no_sync(self):
        """Gradient accumulation (HF `gradient_accumulation_steps`, DDP.no_sync semantics): inside the context, backward only accumulates
        into the local flat gradient buckets; the first backward outside it reduce-scatters the accumulated sum."""
        import contextlib

        @contextlib.contextmanager
        def ctx():
            prev, self._sync = self._sync, False
            try:
                yield
            finally:
                self._sync = prev
                for b in self.buckets:                 # the next backward awaits every parameter again (p.grad stays the bucket view,
                    if not b.launched:                 # so later micro-batches accumulate in place)
                        b.pending = set(b.params)
        return ctx()

    def zero_grad(self, set_to_none: bool = True):
        for b in self.buckets:
            for p in b.params:
                p.grad = None
            b.pending = set(b.params)
            b.seen = set()
            b.ready = b.launched = False
        self._next = 0

    # ------------------------------------------------------------------------------------------ step
    @torch.no_grad()
    def step(self, lr_scale: float = 1.0, defer_gather: bool = False):
        """Finish the gradient reduce-scatters, clip by the global norm, update the owned shards, all-gather the parameters.
        Returns the (unclipped) global gradient norm as a 0-d device tensor (no host sync).
        `defer_gather=True` (needs `attach(model)`): the all-gathers are issued in forward order and only waited for by the forward
        pre-hook of the first module that reads each bucket, so they overlap the start of the next forward instead of ending the step."""
        self.wait_gathers()
        for b in self.buckets:
            for p in b.params:
                if p.data.data_ptr() != b.pviews[p].data_ptr():
                    raise RuntimeError("a parameter was moved out of its optimizer bucket (module.to() / load_state_dict(assign=True) / a "
                                       "weight re-fusion after ShardedAdamW was built); call ShardedAdamW.reseat() after such changes")
        for b in self.buckets[self._next:]:                   # flush in bucket order; a parameter that received no gradient in ANY
            if b.seen or self.world > 1:                      # micro-batch since zero_grad() counts as zero (never discard accumulated ones)
                for p in b.params:
                    if p not in b.seen:
                        b.gviews[p].zero_()
                        p.grad = b.gviews[p]
            self._reduce_scatter(b)
        self._next = len(self.buckets)
        for b in self.buckets:
            if b.work is not None:
                b.work.wait()
                b.work = None
        self.step_count += 1
        clip = self.max_grad_norm > 0
        self._ss.zero_()
        live = [b for b in self.buckets if b.seen or self.world > 1]   # single process, no grad at all in a bucket: skip it (torch skips p.grad None)
        for b in live:
            self._sumsq(b.gshard, self._ss)
        if self.world > 1:
            dist.all_reduce(self._ss, op=dist.ReduceOp.SUM, group=self.pg)
        if defer_gather and not self._attached:
            raise RuntimeError("defer_gather=True needs ShardedAdamW.attach(model) (forward pre-hooks wait for the parameter all-gathers)")
        for b in sorted(live, key=lambda bb: bb.params[0]._zero_order):        # forward order: the first layers' parameters arrive first
            g = b.group
            self._update(b.gshard, b.pshard, b.m, b.v, b.master, lr=g["lr"] * lr_scale, beta1=g["betas"][0], beta2=g["betas"][1],
                         eps=g["eps"], weight_decay=g["weight_decay"], step=self.step_count, grad_sumsq=self._ss if clip else None,
                         max_grad_norm=self.max_grad_norm)
            if self.world > 1:
                b.gather = dist.all_gather_into_tensor(b.flat_param, b.pshard, group=self.pg, async_op=True)
                self.launched += 1
        if not defer_gather:
            self.wait_gathers()
        for b in self.buckets:
            b.pending = set(b.params)
            b.ready = b.launched = False
        self._next = 0
        return self._ss.sqrt().squeeze(0)

    def wait_gathers(self, buckets=None):
        """Make the current stream wait for outstanding parameter all-gathers (all buckets, or the given ones)."""
        for b in (self.buckets if buckets is None else buckets):
            if b.gather is not None:
                b.gather.wait()
                b.gather = None

    def attach(self, model):
        """Register forward pre-hooks on every module that directly owns bucketed parameters: before such a module runs, the all-gathers
        of the buckets it reads are waited for (no-op when none is outstanding).  Enables `step(defer_gather=True)`."""
        for mod in model.modules():
            mine = []
            for p in mod.parameters(recurse=False):
                b = self._bucket_of.get(p)
                if b is not None and b not in mine:
                    mine.append(b)
            if mine:
                self._hooks.append(mod.register_forward_pre_hook(lambda m, args, _b=tuple(mine): self.wait_gathers(_b)))
        self._attached = True
        return self

    # ------------------------------------------------------------------------------------------ checkpoint / resume
    def state_dict(self):
        self.wait_gathers()
        """This rank's shard of the optimizer state (the reference saves FSDP-sharded optimizer state per rank as well)."""
        return {"step": self.step_count, "world": self.world, "rank": self.rank, "state_dtype": str(self.state_dtype),
                "buckets": [{"n": b.n, "chunk": b.chunk, "m": b.m.clone(), "v": b.v.clone(),
                             "master": None if b.master is None else b.master.clone()} for b in self.buckets]}

    def load_state_dict(self, sd):
        if sd["world"] != self.world or sd["rank"] != self.rank or len(sd["buckets"]) != len(self.buckets):
            raise ValueError("optimizer shard was saved for a different world size / rank / bucket layout")
        self.step_count = int(sd["step"])
        for b, s in zip(self.buckets, sd["buckets"]):
            if s["n"] != b.n or s["chunk"] != b.chunk:
                raise ValueError("bucket layout mismatch")
            b.m.copy_(s["m"])
            b.v.copy_(s["v"])
            if b.master is not None:
                b.master.copy_(s["master"])

    def state_bytes_per_rank(self) -> int:
        return sum(t.numel() * t.element_size() for b in self.buckets for t in (b.m, b.v, b.master) if t is not None)

    def remove(self):
        for h in self._hooks:
            h.remove()

"""Bucketed gradient all-reduce overlapped with backward (data-parallel hot path, SURVEY.md §8e).

Replaces what the reference gets implicitly from `DistributedDataParallel` via HF Trainer / accelerate
(omni/train/trainer.py:577-601: `_wrap_model` -> DDP, 25 MB buckets, all-reduce overlapped with backward).
One process per GPU; torch.distributed (NCCL over NVLink/NVSwitch; gloo in the CPU tests) is the transport.

Rules that make it safe when ranks see different batches (stage-2 interleaved data mixes text-only, image and dream samples, so a rank
may produce no gradient for the CLIP projector / dream queries / SD projector in a given step — the reference's "dummy forward" hacks,
modeling_dreamllm.py:1142-1144, :1443-1445, modeling_plugins.py:315-329, exist for exactly that):

* **collectives are issued in bucket-index order on every rank** (torch DDP's in-order rule): a bucket whose gradients are all written is
  only *marked* ready; bucket i is launched once buckets 0..i-1 have been launched, and `finalize()` flushes the rest in index order with
  missing gradients counted as zero.  Every rank therefore issues the same sequence of all-reduces over the same buffers no matter which
  parameters its batch touched.  `late_params` moves parameters that are often unused (plugin projectors, dream queries) to the last
  buckets so that they cannot hold back the overlap of the LLM's buckets.
* **gradients live in the flat buckets**: every parameter carries `_dllm_grad_view` (its slice of the bucket); the wgrad GEMMs of
  `modeling_dreamllm` write straight into it (`ops.linear_wgrad(..., out=view)`) when `p.grad is None`, and autograd then adopts the
  returned alias as `p.grad` — no per-step memset of the buckets and no copy into them.  A gradient produced elsewhere is copied in once.
"""
from __future__ import annotations

import contextlib
import os as _os

import torch
import torch.distributed as dist

NCCL_CTAS = int(_os.environ.get("DLLM_NCCL_CTAS", "0"))        # SM budget handed to the overlapped all-reduce (0 = leave NCCL alone)
RESERVED_SMS = int(_os.environ.get("DLLM_RESERVED_SMS", "0"))  # SMs kept out of the persistent GEMM grids while grads are in flight


def configure_nccl_env():
    """Optional knobs, off by default: NCCL_MAX_CTAS caps the all-reduce's CTAs, reserved SMs keep the persistent GEMM grids off SMs the
    overlapped all-reduce occupies.  Whether either helps on a given multi-GPU H100 box has to be measured there."""
    import os
    if NCCL_CTAS > 0:
        os.environ.setdefault("NCCL_MAX_CTAS", str(NCCL_CTAS))
        os.environ.setdefault("NCCL_MIN_CTAS", "1")


def grad_out_view(params):
    """One tensor covering the bucket gradient slices of `params` (consecutive row blocks of one fused weight, e.g. q|k|v) when a reducer
    / sharded optimizer owns their gradients, every `p.grad` is still None (first write of this step: later micro-batches must go through
    autograd's accumulate) and the slices are adjacent in bucket memory; else None (the caller allocates)."""
    views = []
    for p in params:
        v = getattr(p, "_dllm_grad_view", None)
        if v is None or p.grad is not None:
            return None
        views.append(v)
    ptr = views[0].data_ptr()
    for v in views:
        if v.data_ptr() != ptr or not v.is_contiguous():
            return None
        ptr += v.numel() * v.element_size()
    if len(views) == 1:
        return views[0]
    rows = sum(v.shape[0] for v in views)
    return torch.as_strided(views[0], (rows,) + tuple(views[0].shape[1:]), views[0].stride())


def _glued(p, nxt):
    """True when `p` and the parameter after it (`nxt`, forward order) must share a bucket: the row blocks of one `_fuse_rows` weight, so
    that the fused wgrad can write all of them at once.  q|k|v are tagged (`_dllm_fused_with_prev`, grouped-query attention makes k/v
    narrower than q); gate|up and any other same-shaped neighbouring matrices are glued by shape."""
    return p.dim() == 2 and (getattr(nxt, "_dllm_fused_with_prev", False) or nxt.shape == p.shape)


def plan_runs(params, cap_bytes):
    """Cut `params` (registration = forward order) into runs of at most `cap_bytes`: cut walking BACKWARDS (the order gradients become
    ready), each run laid out in forward order, never between glued neighbours (`_glued`), always where dtype or device changes.  The one
    rule both the gradient reducer and `zero.ShardedAdamW` bucket by."""
    out, run, run_bytes = [], [], 0
    for p in reversed(params):
        nb = p.numel() * p.element_size()
        same = (not run) or (p.dtype == run[0].dtype and p.device == run[0].device)
        if run and (not same or (not _glued(p, run[-1]) and run_bytes + nb > cap_bytes)):
            out.append(list(reversed(run)))
            run, run_bytes = [], 0
        run.append(p)
        run_bytes += nb
    if run:
        out.append(list(reversed(run)))
    return out


def plan_buckets(params, cap_bytes, late=()):
    """`plan_runs` over the parameters in forward order; `late` parameters form the last bucket(s)."""
    late_ids = {id(p) for p in late}
    main = [p for p in params if id(p) not in late_ids]
    tail = [p for p in params if id(p) in late_ids]
    return plan_runs(main, cap_bytes) + plan_runs(tail, cap_bytes)


class BucketedGradReducer:
    def __init__(self, params, bucket_cap_mb: float = 256.0, process_group=None, average: bool = True, late_params=()):
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.average = average
        self.params = [p for p in params if p.requires_grad]
        self.buckets = []           # dict(flat, views{param: view}, params, pending:set, ready, launched, work)
        for plist in plan_buckets(self.params, int(bucket_cap_mb * 1024 * 1024), late=[p for p in late_params if p.requires_grad]):
            self._make_bucket(plist)
        self._bucket_of = {}
        for b in self.buckets:
            for p in b["params"]:
                self._bucket_of[p] = b
        self._hooks = [p.register_post_accumulate_grad_hook(self._on_grad) for p in self.params]
        backend = dist.get_backend(process_group) if dist.is_initialized() else None
        self._use_avg_op = backend == "nccl"
        self.launched = 0
        self.copies = 0             # gradients that had to be copied into their bucket (0 on the fused-wgrad path)
        self._next = 0              # index of the next bucket to launch (in-order rule)
        self._sync = True
        if backend == "nccl" and self.world > 1:
            from ._lib import lib
            lib().dllm_set_reserved_sms(RESERVED_SMS)

    def _make_bucket(self, plist):
        n = sum(p.numel() for p in plist)
        flat = torch.zeros(n, dtype=plist[0].dtype, device=plist[0].device)
        views, off = {}, 0
        for p in plist:
            views[p] = flat[off:off + p.numel()].view_as(p)
            p._dllm_grad_view = views[p]
            off += p.numel()
        self.buckets.append(dict(flat=flat, views=views, params=list(plist), pending=set(plist), seen=set(), ready=False, launched=False,
                                 work=None))

    # called by autograd right after p.grad has been written / accumulated for this backward pass
    def _on_grad(self, p):
        b = self._bucket_of[p]
        v = b["views"][p]
        if p.grad.data_ptr() != v.data_ptr():
            v.copy_(p.grad)
            p.grad = v                    # later micro-batches accumulate in place; the reduced result lands directly in p.grad
            self.copies += 1
        b["seen"].add(p)
        b["pending"].discard(p)
        if not b["pending"] and self._sync:
            b["ready"] = True
            self._launch_ready()

    def _launch_ready(self):
        while self._next < len(self.buckets) and self.buckets[self._next]["ready"]:
            self._launch(self.buckets[self._next])
            self._next += 1

    def _launch(self, b):
        b["launched"] = True
        if self.world == 1:
            return
        flat = b["flat"]
        if self._use_avg_op and self.average:
            b["work"] = dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=self.group, async_op=True)
        else:
            if self.average:
                flat.div_(self.world)
            b["work"] = dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
        self.launched += 1

    def no_sync(self):
        """Gradient accumulation (DDP.no_sync): backward inside the context only accumulates into the bucket views; the first backward
        outside it (or `finalize()`) reduces the accumulated sum."""
        @contextlib.contextmanager
        def ctx():
            prev, self._sync = self._sync, False
            try:
                yield
            finally:
                self._sync = prev
                for b in self.buckets:                       # next micro-batch: every parameter is awaited again
                    if not b["launched"]:
                        b["pending"] = set(b["params"])
        return ctx()

    def finalize(self):
        """Call after the (last) backward: flush, in index order, the buckets not launched yet — parameters that received no gradient
        since `zero_grad()` count as zero — and wait for every all-reduce."""
        for b in self.buckets[self._next:]:
            for p in b["params"]:
                if p not in b["seen"]:
                    b["views"][p].zero_()
                    p.grad = b["views"][p]
            self._launch(b)
        self._next = len(self.buckets)
        for b in self.buckets:
            if b["work"] is not None:
                b["work"].wait()
                b["work"] = None

    def zero_grad(self):
        """Start a new step.  `p.grad = None` (not a memset): the first gradient of the step overwrites the parameter's bucket slice —
        written there directly by the fused wgrad GEMMs, or copied in once by the hook."""
        for b in self.buckets:
            for p in b["params"]:
                p.grad = None
            b["pending"] = set(b["params"])
            b["seen"] = set()
            b["ready"] = b["launched"] = False
        self._next = 0

    def remove(self):
        for h in self._hooks:
            h.remove()
        for p in self.params:
            if hasattr(p, "_dllm_grad_view"):
                del p._dllm_grad_view

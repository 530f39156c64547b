"""CPU tests of packed (unpadded) batches: `DataCollatorForDreamLLMDataset(pack=True)`, the host-side validation of `cu_seqlens`, and
the C-ABI entries of the variable-length attention kernels.

A packed batch is the right-padded batch with the pad positions deleted, so every check here is against `pack=False` on the same
examples (whose output is pinned to the reference collator by test_collator_cpu.py).
"""
import ctypes
import os
import re
from types import SimpleNamespace

import pytest
import torch

from dreamllm_b200.collator import DataCollatorForDreamLLMDataset, to_device

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAD, IM_START, IM_PATCH, IM_END, DREAM_START, DREAM_END = 0, 500, 501, 502, 503, 504
P, Q, H = 6, 4, 8
TOK = SimpleNamespace(pad_token_id=PAD)


def _sample(g, n_text, image=False, dream=False, extra_im_start=False):
    ids, lab = [1], [-100]
    if image:
        ids += [IM_START] + [IM_PATCH] * P + [IM_END]
        lab += [-100] * (P + 2)
    t = torch.randint(5, 400, (n_text,), generator=g).tolist()
    ids += t
    lab += t
    if extra_im_start:                      # an <im_start> with no image behind it stays a token embedding
        ids += [IM_START] + [IM_PATCH] * P + [IM_END]
        lab += [-100] * (P + 2)
    if dream:
        ids += [DREAM_START] + [IM_PATCH] * Q + [DREAM_END]
        lab += [-100] * (Q + 2)
    ids.append(2)
    lab.append(2)
    return dict(input_ids=torch.tensor(ids), attention_mask=torch.ones(len(ids), dtype=torch.long), labels=torch.tensor(lab),
                images=torch.randn(1, 3, 4, 4, generator=g) if image else None,
                images_dm=torch.randn(1, 3, 8, 8, generator=g) if dream else None)


def _collator(**kw):
    return DataCollatorForDreamLLMDataset(TOK, image_start_id=IM_START, dream_start_id=DREAM_START, clip_embed_len=P, dream_embed_len=Q, **kw)


def _batch(seed=0):
    """images + dream queries, an image with a surplus <im_start>, a dream only, a sample with neither; four different lengths"""
    g = torch.Generator().manual_seed(seed)
    return [_sample(g, 11, image=True, dream=True), _sample(g, 3, image=True, extra_im_start=True), _sample(g, 17, dream=True),
            _sample(g, 5)]


@pytest.mark.parametrize("seed", [0, 1])
def test_packed_batch_is_the_padded_batch_without_its_pad_positions(seed):
    ex = _batch(seed)
    pad, pk = _collator()(ex), _collator(pack=True)(ex)
    valid = pad["attention_mask"].bool()
    lens = pad["seqlens"]
    T = int(lens.sum())
    for k in ("input_ids", "labels", "shifted_labels", "attention_mask", "position_ids"):
        assert pk[k].shape == (1, T), k
    assert torch.equal(pk["input_ids"][0], pad["input_ids"][valid])          # boolean indexing walks the batch in row-major order
    assert torch.equal(pk["labels"][0], pad["labels"][valid])
    assert bool((pk["attention_mask"] == 1).all()) and pk["attention_mask_has_padding"] is False
    assert pk["cu_seqlens"].dtype == torch.int32 and pk["cu_seqlens"].tolist() == [0] + torch.cumsum(lens, 0).tolist()
    assert torch.equal(pk["seqlens"], lens) and pk["max_seqlen"] == int(lens.max()) and isinstance(pk["max_seqlen"], int)
    assert pk["position_ids"][0].tolist() == [i for n in lens.tolist() for i in range(n)]
    # the shift never crosses a boundary: the padded shift at the valid positions, -100 at every sample's last token
    assert torch.equal(pk["shifted_labels"][0], pad["shifted_labels"][valid])
    last = pk["cu_seqlens"][1:].long() - 1
    assert bool((pk["shifted_labels"][0, last] == -100).all())
    assert pk["num_label_tokens"] == pad["num_label_tokens"] and pk["num_tokens"] == pad["num_tokens"] == T
    assert pk["input_ids_cpu"] is pk["input_ids"]
    for k in ("images", "images_dm"):
        assert torch.equal(pk[k], pad[k])
    moved = to_device(pk, "cpu")
    assert moved["max_seqlen"] == pk["max_seqlen"] and moved["cu_seqlens"] is pk["cu_seqlens"]      # both stay on the host


def test_unpacked_output_is_unchanged():
    """`pack=False` (the default) emits exactly the keys and values it always did: the reference collator's, plus the index maps."""
    ex = _batch()
    got = _collator()(ex)
    assert set(got) == {"input_ids", "attention_mask", "labels", "images", "images_dm", "input_ids_cpu", "splice_plan",
                        "attention_mask_has_padding", "seqlens", "cu_seqlens", "shifted_labels", "num_tokens", "num_label_tokens"}
    pad = torch.nn.utils.rnn.pad_sequence
    assert torch.equal(got["input_ids"], pad([e["input_ids"] for e in ex], batch_first=True, padding_value=PAD))
    assert torch.equal(got["labels"], pad([e["labels"] for e in ex], batch_first=True, padding_value=-100))
    assert torch.equal(got["attention_mask"], pad([e["attention_mask"] for e in ex], batch_first=True, padding_value=0))
    assert got["attention_mask_has_padding"] is True and to_device(got, "cpu")["cu_seqlens"] is not None


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_packed_splice_plan_addresses_the_same_tokens(seed):
    ex = _batch(seed)
    pad, pk = _collator()(ex), _collator(pack=True)(ex)
    S = pad["input_ids"].shape[1]
    cu = pk["cu_seqlens"].long()

    def remap(rows):                     # row b * S + s of the padded rectangle -> row cu[b] + s of the packed sequence
        rows = rows.long()
        return cu[rows // S] + rows % S

    a, b = pad["splice_plan"], pk["splice_plan"]
    for f in ("img_dst", "dq_dst", "dq_rows", "cond_rows"):
        assert torch.equal(remap(getattr(a, f)), getattr(b, f).long()), f
        assert getattr(b, f).dtype == torch.int32
    for f in ("img_src", "dq_src", "dq_seg"):
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    assert (a.n_images_used, a.n_dreams) == (b.n_images_used, b.n_dreams) == (2, 2)
    text_only = _collator(pack=True)([ex[3], ex[3]])
    assert text_only["splice_plan"] is None and text_only["cu_seqlens"].tolist() == [0, 7, 14]


def test_a_span_that_runs_over_a_sample_boundary_is_rejected():
    """Over [1, T] ids a truncated image span would run on into the next sample unnoticed by the plan builder (it bounds a span by the
    row length, which is T), so the packed collator bounds it by the sample."""
    g = torch.Generator().manual_seed(3)
    cut = _sample(g, 4, image=True)
    keep = 1 + 1 + P - 2                  # bos, <im_start> and all but two of its patch positions
    cut = {k: (v[:keep] if k in ("input_ids", "attention_mask", "labels") else v) for k, v in cut.items()}
    with pytest.raises(ValueError, match="past the end of its sample"):
        _collator(pack=True)([cut, _sample(g, 9)])
    with pytest.raises(ValueError, match="past the end of its sample"):
        dream = _sample(g, 4, dream=True)
        dream = {k: (v[:-3] if k in ("input_ids", "attention_mask", "labels") else v) for k, v in dream.items()}
        _collator(pack=True)([dream, _sample(g, 9)])


def test_cu_seqlens_is_validated_on_the_host():
    from dreamllm_b200.modeling_dreamllm import _packed_batch
    cu, ms = _packed_batch(torch.tensor([0, 3, 3, 10], dtype=torch.int32), 7, 10, "cpu")
    assert cu.dtype == torch.int32 and cu.tolist() == [0, 3, 3, 10] and ms == 7
    assert _packed_batch(torch.tensor([0, 3, 10]), 8, 10, "cpu")[1] == 8
    for bad, ms, msg in (([0, 3, 9], 7, "number of packed tokens"), ([1, 3, 10], 7, "number of packed tokens"),
                         ([0, 6, 4, 10], 6, "non-decreasing"), ([0, 3, 10], 6, "max_seqlen"), ([0, 3, 10], 11, "max_seqlen")):
        with pytest.raises(ValueError, match=msg):
            _packed_batch(torch.tensor(bad, dtype=torch.int32), ms, 10, "cpu")
    with pytest.raises(ValueError, match="1-D"):
        _packed_batch(torch.tensor([10]), 10, 10, "cpu")


def test_varlen_entries_are_exported_with_the_declared_signatures():
    from dreamllm_b200 import _lib
    _lib.build()
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "dreamllm_sm100.h")).read()
    ctype = {"int": ctypes.c_int, "long": ctypes.c_long, "float": ctypes.c_float, "size_t": ctypes.c_size_t}
    for name in ("dllm_attn_fwd_varlen", "dllm_attn_bwd_varlen_workspace_bytes", "dllm_attn_bwd_varlen"):
        assert hasattr(L, name), name
        m = re.search(r"\b(int|size_t)\s+" + name + r"\s*\(([^;]*)\);", hdr)
        assert m, f"{name} is not declared in the header"
        args = [a.strip() for a in m.group(2).replace("\n", " ").split(",")]
        want = [ctypes.c_void_p if "*" in a else ctype[a.split()[0]] for a in args]
        res, got = _lib.SIGNATURES[name]
        assert res is ctype[m.group(1)] and got == want, (name, args)
    # host query: two fp32 planes [nh, round_up(T, 64) + 64]
    assert L.dllm_attn_bwd_varlen_workspace_bytes(4248, 32, 128) == (4288 + 64) * 32 * 2 * 4
    assert L.dllm_attn_bwd_varlen_workspace_bytes(64, 2, 64) == 128 * 2 * 2 * 4

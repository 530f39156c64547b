"""Batch collator that emits the device index maps of the hot path (SURVEY.md §8f row 3).

Drop-in for `DataCollatorForDreamLLMDataset` (omni/data/builders/builder_dreamllm.py:467-482): same constructor field (`tokenizer`),
same `__call__(examples: list[dict]) -> dict`, same keys with the same values (`input_ids`, `attention_mask`, `labels` right-padded with
`pad_token_id` / 0 / -100; `images`, `images_dm` concatenated or None).  On top of those it emits everything the reference's forward
derives from `input_ids` with host syncs every step (`torch.where` per sample, `0 in attention_mask`, modeling_dreamllm.py:962,
:1082-1141, :1401-1418), computed here once, on the host, in the dataloader worker:

    input_ids_cpu               the padded ids, kept on the host (no D2H copy in forward)
    splice_plan                 `SplicePlan` (host, int32): scatter maps for image features / dream queries, the CSR map for the dream
                                query gradient, the conditioning gather rows — moved to the GPU with `SplicePlan.to(device)`
    attention_mask_has_padding  bool: replaces `0 in attention_mask`
    seqlens                     int32 [B] valid lengths (what the attention kernels take), `cu_seqlens` int32 [B+1]
    shifted_labels              int64 [B, S]: labels[:, 1:] with -100 in the last column (the shift of :1456-1459 done once)
    num_tokens / num_label_tokens  python ints for throughput / loss bookkeeping (the bench's tokens-per-step)

`DreamLLMForCausalMLM.forward(**batch)` accepts these keys directly (`splice_plan`, `input_ids_cpu`, `attention_mask_has_padding`).

`pack=True` emits the same keys for a packed (unpadded) batch instead: the samples' tokens laid end to end as one row of T =
sum(len_b) tokens, so that no kernel of the step computes a pad row.  `input_ids` / `labels` / `attention_mask` (all ones) /
`position_ids` (restarting at 0 in every sample) / `shifted_labels` are [1, T]; `cu_seqlens` int32 [B + 1] says where each sample
starts, `max_seqlen` (python int) is the longest one; `shifted_labels` is -100 at the last token of every sample, so no label crosses
a boundary; the splice plan addresses rows of the packed sequence.
Pure host integer work: no CUDA, no kernels; safe in worker processes.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import torch

from .modeling_plugins import SplicePlan, build_splice_plan

IGNORE_INDEX = -100


def _pad(seqs, value):
    return torch.nn.utils.rnn.pad_sequence(list(seqs), batch_first=True, padding_value=value)


@dataclass
class DataCollatorForDreamLLMDataset:
    tokenizer: object                       # needs `.pad_token_id` (reference: PreTrainedTokenizerBase)
    image_start_id: int = -1                # <im_start> id  (special_tokens2ids_dict["additional_special_tokens"]["<im_start>"])
    dream_start_id: int = -1                # <dream_start> id
    clip_embed_len: int = 0                 # P = clip_vision_embedding.embed_len (train.py:185-188 reads the same attribute)
    dream_embed_len: int = 0                # Q = dream_embedding.embed_len
    pin_memory: bool = False                # pin the index maps (set in the main process; workers cannot pin)
    pad_to_multiple_of: int | None = None   # optional: round S up (keeps TMA tiles full); reference pads to the batch max only
    extra_keys: tuple = field(default_factory=tuple)
    pack: bool = False                      # emit one packed [1, T] row + cu_seqlens instead of the right-padded [B, S] rectangle

    @classmethod
    def from_model(cls, tokenizer, model, **kw):
        """Read the ids and embed lengths off a DreamLLMForCausalMLM the way the dataset builder does (train.py:185-188)."""
        m = model.model
        clip = getattr(m, "clip_vision_embedding", None)
        dream = getattr(m, "dream_embedding", None)
        return cls(tokenizer, image_start_id=getattr(m, "image_start_id", None) if clip is not None else -1,
                   dream_start_id=getattr(m, "dream_start_id", None) if dream is not None else -1,
                   clip_embed_len=clip.embed_len if clip is not None else 0, dream_embed_len=dream.embed_len if dream is not None else 0, **kw)

    def __call__(self, examples: list[dict]) -> dict:
        keys = examples[0].keys()
        batch = {k: [e[k] for e in examples] for k in keys}
        pad_id = self.tokenizer.pad_token_id
        ids = _pad(batch["input_ids"], pad_id)
        mask = _pad(batch["attention_mask"], 0)
        labels = _pad(batch["labels"], IGNORE_INDEX)
        if self.pad_to_multiple_of:
            S = ids.shape[1]
            S2 = (S + self.pad_to_multiple_of - 1) // self.pad_to_multiple_of * self.pad_to_multiple_of
            if S2 != S:
                ids = torch.nn.functional.pad(ids, (0, S2 - S), value=pad_id)
                mask = torch.nn.functional.pad(mask, (0, S2 - S), value=0)
                labels = torch.nn.functional.pad(labels, (0, S2 - S), value=IGNORE_INDEX)
        images = [x for x in batch.get("images", []) if x is not None]
        images = torch.cat(images, 0) if len(images) > 0 else None
        images_dm = [x for x in batch.get("images_dm", []) if x is not None]
        images_dm = torch.cat(images_dm, 0) if len(images_dm) > 0 else None
        out = dict(batch)
        out.update(input_ids=ids, attention_mask=mask, labels=labels, images=images, images_dm=images_dm)
        if "add_time_ids" in batch:
            # SDXL micro-conditioning: [n, 6] per example, concatenated in batch order, None if no example has any
            # (reference builder_dreamllm.py:452-453, :501-502)
            add_time_ids = [torch.as_tensor(x).reshape(-1, 6) for x in batch["add_time_ids"] if x is not None]
            out["add_time_ids"] = torch.cat(add_time_ids, 0) if len(add_time_ids) > 0 else None

        # ---- device index maps (the part the reference recomputes on the GPU with host syncs every step)
        seqlens = mask.sum(-1).to(torch.int32)
        right_padded = bool((mask == (torch.arange(mask.shape[1])[None] < seqlens[:, None])).all())
        if not right_padded:
            raise ValueError("attention_mask is not a right-padded prefix mask (the collator pads on the right, builder_dreamllm.py:470-472)")
        if self.pack:
            out.update(self._packed(ids, labels, seqlens, images, images_dm))
            return out
        plan = None
        if images is not None or images_dm is not None:
            plan = build_splice_plan(ids, self.image_start_id if images is not None else -1,
                                     self.dream_start_id if images_dm is not None else -1,
                                     self.clip_embed_len if images is not None else 0, self.dream_embed_len if images_dm is not None else 0,
                                     0 if images is None else images.shape[0], None if images_dm is None else images_dm.shape[0], "cpu")
            if self.pin_memory:
                plan = plan.pin_memory()
        shifted = torch.full_like(labels, IGNORE_INDEX)
        shifted[:, :-1] = labels[:, 1:]
        cu = torch.zeros(ids.shape[0] + 1, dtype=torch.int32)
        cu[1:] = torch.cumsum(seqlens, 0)
        out.update(input_ids_cpu=ids, splice_plan=plan, attention_mask_has_padding=bool((seqlens < ids.shape[1]).any()),
                   seqlens=seqlens, cu_seqlens=cu, shifted_labels=shifted, num_tokens=int(seqlens.sum()),
                   num_label_tokens=int((shifted != IGNORE_INDEX).sum()))
        return out

    def _packed(self, ids, labels, seqlens, images, images_dm) -> dict:
        """The packed form of the right-padded `ids` / `labels` [B, S]: their valid prefixes, in batch order, as one [1, T] row."""
        B, S = ids.shape
        valid = torch.arange(S)[None] < seqlens[:, None]
        cu = torch.zeros(B + 1, dtype=torch.int32)
        cu[1:] = torch.cumsum(seqlens, 0)
        T = int(cu[-1])
        if T == 0:
            raise ValueError("cannot pack a batch without a single token")
        shifted = torch.full_like(labels, IGNORE_INDEX)
        shifted[:, :-1] = labels[:, 1:]                    # the pad column after a sample's last token is already -100
        shifted[torch.arange(B), (seqlens.long() - 1).clamp_(min=0)] = IGNORE_INDEX
        pids = ids[valid][None]
        plan = None
        if images is not None or images_dm is not None:
            P = self.clip_embed_len if images is not None else 0
            Q = self.dream_embed_len if images_dm is not None else 0
            img_id = self.image_start_id if images is not None else -1
            dream_id = self.dream_start_id if images_dm is not None else -1
            # build_splice_plan bounds a span by its row's length, which for [1, T] ids is T: bound it by its own sample here
            room = (seqlens[:, None] - 1 - torch.arange(S)[None])[valid]        # tokens after each position, inside its sample
            n_img = 0 if images is None else images.shape[0]
            img_at = (pids[0] == img_id).nonzero()[:n_img, 0]
            dream_at = (pids[0] == dream_id).nonzero()[:, 0]
            if bool((room[img_at] < P).any()) or bool((room[dream_at] < Q).any()):
                raise ValueError("an image / dream-query span runs past the end of its sample (reference assert :1126)")
            plan = build_splice_plan(pids, img_id, dream_id, P, Q, n_img, None if images_dm is None else images_dm.shape[0], "cpu")
            if self.pin_memory:
                plan = plan.pin_memory()
        pos = (torch.arange(S)[None].expand(B, S))[valid][None]
        pshift = shifted[valid][None]
        return dict(input_ids=pids, attention_mask=torch.ones_like(pids), labels=labels[valid][None], position_ids=pos,
                    input_ids_cpu=pids, splice_plan=plan, attention_mask_has_padding=False, seqlens=seqlens, cu_seqlens=cu,
                    max_seqlen=int(seqlens.max()), shifted_labels=pshift, num_tokens=T,
                    num_label_tokens=int((pshift != IGNORE_INDEX).sum()))


def to_device(batch: dict, device, non_blocking: bool = True) -> dict:
    """Move a collated batch to the GPU with async copies only (host-side keys stay on the host).  A packed batch keeps `max_seqlen`
    and `cu_seqlens` on the host: the model validates the boundaries there, without a device read-back, and uploads them itself."""
    out = {}
    packed = "max_seqlen" in batch
    for k, v in batch.items():
        if packed and k == "cu_seqlens":
            out[k] = v
            continue
        if k == "input_ids_cpu" or k in ("num_tokens", "num_label_tokens", "attention_mask_has_padding", "max_seqlen"):
            out[k] = v
        elif isinstance(v, SplicePlan):
            out[k] = v.to(device, non_blocking=non_blocking)
        elif torch.is_tensor(v):
            out[k] = v.to(device, non_blocking=non_blocking)
        else:
            out[k] = v
    return out

"""Token sampling for `DreamLLMForCausalMLM.generate` (SURVEY.md §8f row 2: the kv-cache decode path the reference reaches through HF
`GenerationMixin.generate`, omni/eval/vqa/vqa_inference.py:112-130, modeling_dreamllm.py:1511-1547).

The per-token model work (prefill + cached decode) is the CUDA path in modeling_dreamllm.py; what lives here is the [B, V] logits
post-processing of one step — the semantics of transformers' `RepetitionPenaltyLogitsProcessor`, `TemperatureLogitsWarper`,
`TopKLogitsWarper`, `TopPLogitsWarper` in HF's order — as a handful of torch ops on the device holding the logits (plumbing, not a hot
path: 32 008 floats per sequence per token).  Greedy (`do_sample=False`) is a plain argmax: bit-exact token ids.
tests/test_generation_cpu.py pins `warp_logits` to the installed transformers processors.
"""
from __future__ import annotations

import torch


def warp_logits(logits: torch.Tensor, input_ids: torch.Tensor | None = None, temperature: float = 1.0, top_k: int = 0,
                top_p: float = 1.0, repetition_penalty: float = 1.0, min_tokens_to_keep: int = 1) -> torch.Tensor:
    """[B, V] fp32 scores -> filtered scores (-inf = removed), HF order: repetition penalty, temperature, top-k, top-p."""
    scores = logits.float()
    if repetition_penalty != 1.0 and input_ids is not None:
        picked = torch.gather(scores, 1, input_ids)
        picked = torch.where(picked < 0, picked * repetition_penalty, picked / repetition_penalty)
        scores = scores.scatter(1, input_ids, picked)
    if temperature != 1.0:
        if not temperature > 0:
            raise ValueError(f"`temperature` has to be a strictly positive float, but is {temperature}")
        scores = scores / temperature
    if top_k and top_k > 0:
        k = min(max(top_k, min_tokens_to_keep), scores.shape[-1])
        kth = torch.topk(scores, k)[0][..., -1, None]
        scores = scores.masked_fill(scores < kth, float("-inf"))
    if top_p is not None and top_p < 1.0:
        if not 0 <= top_p <= 1.0:
            raise ValueError(f"`top_p` has to be a float > 0 and < 1, but is {top_p}")
        sorted_logits, sorted_indices = torch.sort(scores, descending=False)
        cumulative_probs = sorted_logits.softmax(dim=-1).cumsum(dim=-1)
        sorted_remove = cumulative_probs <= (1 - top_p)
        sorted_remove[..., -min_tokens_to_keep:] = False
        remove = sorted_remove.scatter(1, sorted_indices, sorted_remove)
        scores = scores.masked_fill(remove, float("-inf"))
    return scores


def pick_next_token(logits: torch.Tensor, input_ids: torch.Tensor | None = None, do_sample: bool = False, generator=None, **warp) -> torch.Tensor:
    """One decoding step over [B, V] logits -> [B] token ids."""
    if not do_sample:
        if warp.get("repetition_penalty", 1.0) != 1.0:
            logits = warp_logits(logits, input_ids, repetition_penalty=warp["repetition_penalty"])
        return logits.argmax(-1)
    probs = warp_logits(logits, input_ids, **warp).softmax(-1)
    return torch.multinomial(probs, 1, generator=generator).squeeze(1)


def ragged(decode_one, input_ids, attention_mask, pad_id: int):
    """Row-by-row fallback for RIGHT-padded prompt batches (pads between the prompt and the new tokens; HF itself warns against that layout
    for decoder-only generation): run `decode_one(ids [1, L])` on every row's valid tokens and lay the result out as HF `generate` does —
    `[original padded prompt row | generated tokens | pad]`, i.e. `out[:, :S] == input_ids` and `out[:, S:]` holds only new tokens (the
    slice `vqa_inference.py` decodes), whatever side the prompt was padded on and however many tokens each row produced."""
    mask = attention_mask.bool()
    S = input_ids.shape[1]
    gens = []
    for row, m in zip(input_ids, mask):
        n_valid = int(m.sum())
        gens.append(decode_one(row[m][None])[0][n_valid:])
    width = max(g.numel() for g in gens)
    out = torch.full((input_ids.shape[0], S + width), pad_id, dtype=input_ids.dtype, device=input_ids.device)
    out[:, :S] = input_ids
    for b, g in enumerate(gens):
        out[b, S:S + g.numel()] = g
    return out


def check_graph_decode(model):
    """Refuse, before the prefill, what the captured decode step does not compute."""
    cfg = model.config
    if getattr(cfg, "output_attentions", False) or getattr(cfg, "log_attentions", False):
        raise ValueError("output_attentions / log_attentions are not available with use_cuda_graph=True: the captured decode step does "
                         "not compute attention probabilities")


def _left_padded(attention_mask) -> bool:
    """True when every row's LAST prompt position is a real token (left padding, or no padding): the batched kv-cache path applies."""
    return bool(attention_mask[:, -1].all())


def _positions(attention_mask):
    """reference `prepare_inputs_for_generation`, :1521-1526: position = number of real tokens before it; pad positions get 1."""
    pos = attention_mask.long().cumsum(-1) - 1
    return pos.masked_fill(attention_mask == 0, 1)


@torch.no_grad()
def generate(model, input_ids, images=None, max_new_tokens: int = 16, do_sample: bool = False, temperature: float = 1.0, top_k: int = 0,
             top_p: float = 1.0, repetition_penalty: float = 1.0, eos_token_id=None, pad_token_id=None, generator=None,
             attention_mask=None, stopping_criteria=None, use_cuda_graph: bool = False):
    """Prefill once with the kv-cache, then one cached decode step per token.  `use_cuda_graph=True` runs every decode step as one
    replay of a captured graph (`decode.DecodeGraph`); the prefill and the token selection are unchanged, the logits differ from the
    eager steps' only in the summation order of the attention.  Finished rows keep emitting `pad_token_id` (HF semantics);
    stops when every row has produced an EOS or a `stopping_criteria` callable `(input_ids, scores) -> bool | BoolTensor[B]` fires for it
    (HF `StoppingCriteria` semantics; the reference's VQA eval passes a keyword criterion, omni/eval/vqa/vqa_inference.py:105-106).
    Returns [B, S + n_generated] ids (prompt included, like HF for decoder-only models)."""
    am = None
    if attention_mask is not None and not bool(attention_mask.all()):
        am = attention_mask.to(input_ids.device)
    if am is not None and not _left_padded(am):
        # right-padded batch: pads would sit between the prompt and the new tokens — each prompt is decoded on its own (batch 1)
        if images is not None:
            raise NotImplementedError("right-padded prompt batches with images: left-pad them (HF's convention for decoder-only models) or "
                                      "pass the prompts one at a time (images are matched to <im_start> tokens in batch order)")
        return ragged(lambda ids: generate(model, ids, None, max_new_tokens, do_sample, temperature, top_k, top_p, repetition_penalty,
                                           eos_token_id, pad_token_id, generator, None, stopping_criteria, use_cuda_graph),
                      input_ids, attention_mask, pad_token_id if pad_token_id is not None else
                      (eos_token_id if isinstance(eos_token_id, int) else (eos_token_id[0] if eos_token_id else 0)))
    eos = None
    if eos_token_id is not None:
        eos = torch.as_tensor([eos_token_id] if isinstance(eos_token_id, int) else list(eos_token_id), device=input_ids.device)
        if pad_token_id is None:
            pad_token_id = int(eos[0])
    if stopping_criteria and pad_token_id is None:
        pad_token_id = 0
    warp = dict(temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty)
    seq = input_ids
    unfinished = torch.ones(input_ids.shape[0], dtype=torch.bool, device=input_ids.device)
    # left-padded batch: ONE batched prefill + batched decode steps; the pad keys stay masked inside the kv-cache and RoPE positions come
    # from the mask, exactly as HF generate drives the reference (vqa_inference.py:112-130, modeling_dreamllm.py:1511-1547)
    mask_kw = {} if am is None else dict(attention_mask=am, position_ids=_positions(am))
    if use_cuda_graph:
        check_graph_decode(model)
    out = model(input_ids=input_ids, images=images, use_cache=True, last_token_logits_only=True, **mask_kw)
    cache = out.past_key_values
    logits = out.logits[:, -1]
    graph = None
    if use_cuda_graph:
        from .decode import DecodeGraph
        graph = DecodeGraph(model, cache, input_ids.shape[0], positions=None if am is None else am.long().sum(-1))
    for i in range(max_new_tokens):
        nxt = pick_next_token(logits, seq, do_sample=do_sample, generator=generator, **warp)
        if pad_token_id is not None:
            nxt = torch.where(unfinished, nxt, torch.full_like(nxt, pad_token_id))       # finished rows keep emitting pad
        if eos is not None:
            unfinished = unfinished & ~torch.isin(nxt, eos)
        seq = torch.cat([seq, nxt[:, None]], 1)
        for crit in (stopping_criteria or ()):
            done = crit(seq, logits)
            done = torch.as_tensor(done, device=seq.device, dtype=torch.bool)
            unfinished = unfinished & ~(done.expand_as(unfinished))
        if i + 1 == max_new_tokens or ((eos is not None or stopping_criteria) and not bool(unfinished.any())):
            break
        if graph is not None:
            graph.ids.copy_(nxt)
            logits = graph.replay()
            continue
        if am is not None:
            am = torch.cat([am, torch.ones_like(am[:, :1])], 1)
            mask_kw = dict(attention_mask=am, position_ids=am.long().sum(-1, keepdim=True) - 1)
        out = model(input_ids=nxt[:, None], past_key_values=cache, use_cache=True, last_token_logits_only=True, **mask_kw)
        logits = out.logits[:, -1]
    return seq


# ------------------------------------------------------------------------------------------------ beam search
def _gather_beams(t: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """t [B, K, ...], idx [B, k] -> t[b, idx[b, j], ...]"""
    view = idx.reshape(idx.shape + (1,) * (t.dim() - 2)).expand(idx.shape + t.shape[2:])
    return torch.gather(t, 1, view)


@torch.no_grad()
def beam_search(model, input_ids, images=None, num_beams: int = 5, max_new_tokens: int = 16, length_penalty: float = 1.0,
                early_stopping=False, eos_token_id=None, pad_token_id=None, stopping_criteria=None,
                length_normalization: str = "generated", return_scores: bool = False, attention_mask=None, use_cuda_graph: bool = False):
    """Beam search over the kv-cache decode path — what `model.generate(..., num_beams=5)` does in the reference's default VQA eval
    (omni/eval/vqa/vqa_inference.py:111-119, `--beamsearch True` is the default, omni/utils/eval_utils.py:141).

    Semantics = transformers' beam search (accumulated log-probs, top `2 x num_beams` continuations per step so that `num_beams` live beams
    survive EOS picks, finished hypotheses ranked by sum_logprobs / length**length_penalty, the `early_stopping=False` "can the best live
    beam still beat the worst finished one" heuristic).  `length_normalization="generated"` divides by the number of generated tokens, as
    transformers >= 4.36 and the version installed here do — tests/test_generation_cpu.py pins this mode to the installed
    `GenerationMixin.generate(num_beams=...)` on random LLaMAs; `"total"` divides by prompt + generated length, the rule of the 4.35.x
    scorer the reference pins (restated from memory: that version cannot be installed here, so this mode is unpinned).
    The prompt is prefilled once per sample; the cache is then repeated per beam and re-ordered in place every step.
    `use_cuda_graph=True` runs the decode steps as replays of one captured graph (`decode.DecodeGraph`), as in `generate`.
    Returns [B, prompt + generated] ids of the best hypothesis per sample (padded with `pad_token_id` after EOS)."""
    if length_normalization not in ("generated", "total"):
        raise ValueError("length_normalization must be 'generated' or 'total'")
    dev = input_ids.device
    B, prompt_len = input_ids.shape
    k = int(num_beams)
    max_length = prompt_len + int(max_new_tokens)
    eos = None
    if eos_token_id is not None:
        eos = torch.as_tensor([eos_token_id] if isinstance(eos_token_id, int) else list(eos_token_id), device=dev)
    n_eos = 0 if eos is None else int(eos.numel())
    K = max(2, 1 + n_eos) * k                                           # candidates kept per sample and step
    fill = pad_token_id if pad_token_id is not None else (int(eos[0]) if eos is not None else 0)
    NEG = -1.0e9

    running = torch.full((B, k, max_length), fill, dtype=torch.long, device=dev)
    running[:, :, :prompt_len] = input_ids[:, None, :]
    finished = running.clone()
    running_scores = torch.zeros((B, k), dtype=torch.float32, device=dev)
    running_scores[:, 1:] = NEG                                         # all beams start identical: only beam 0 may branch
    finished_scores = torch.full((B, k), NEG, dtype=torch.float32, device=dev)
    finished_len = torch.zeros((B, k), dtype=torch.long, device=dev)    # generated tokens of each finished hypothesis
    is_finished = torch.zeros((B, k), dtype=torch.bool, device=dev)
    heuristic_open = torch.ones((B, 1), dtype=torch.bool, device=dev)
    top_k_mask = torch.arange(K, device=dev)[None, :] < k

    def norm_len(generated):                                             # length used by the length penalty
        return float(generated if length_normalization == "generated" else generated + prompt_len)

    am = None                                                            # left-padded prompt batch: pad keys masked inside the cache
    if attention_mask is not None and not bool(attention_mask.all()):
        am = attention_mask.to(dev)
        if not _left_padded(am):
            raise ValueError("beam search over a padded batch needs LEFT padding (HF's convention for decoder-only models)")
    mask_kw = {} if am is None else dict(attention_mask=am, position_ids=_positions(am))
    if use_cuda_graph:
        check_graph_decode(model)
    out = model(input_ids=input_ids, images=images, use_cache=True, last_token_logits_only=True, **mask_kw)
    cache = out.past_key_values
    cache.repeat_interleave(k)
    if am is not None:
        am = am.repeat_interleave(k, dim=0)
    graph = None
    if use_cuda_graph:                                                   # built after repeat_interleave, which reallocates the cache
        from .decode import DecodeGraph
        graph = DecodeGraph(model, cache, B * k, positions=None if am is None else am.long().sum(-1))
    logits = out.logits[:, -1].float().repeat_interleave(k, dim=0)      # [B*k, V]
    cur_len = prompt_len
    while True:
        V = logits.shape[-1]
        logp = torch.log_softmax(logits, dim=-1).view(B, k, V) + running_scores[:, :, None]
        cand_scores, flat = torch.topk(logp.view(B, k * V), K, dim=1)
        src_beam, token = flat // V, flat % V
        cand = _gather_beams(running, src_beam)
        cand[:, :, cur_len] = token
        hits = torch.zeros((B, K), dtype=torch.bool, device=dev)
        if eos is not None:
            hits |= torch.isin(token, eos)
        if cur_len + 1 >= max_length:
            hits |= True
        for crit in (stopping_criteria or ()):                       # HF StoppingCriteria: (candidate sequences [B*K, len], scores) -> bool | [B*K]
            done = torch.as_tensor(crit(cand[:, :, :cur_len + 1].reshape(B * K, cur_len + 1), None), device=dev, dtype=torch.bool)
            hits |= done.reshape(B, K) if done.numel() == B * K else bool(done)
        # live beams for the next step: the best num_beams candidates that did not just finish
        live_scores = cand_scores + hits.float() * NEG
        pick = torch.topk(live_scores, k, dim=1)[1]
        running = _gather_beams(cand, pick)
        running_scores = _gather_beams(live_scores, pick)
        next_src = _gather_beams(src_beam, pick)
        # finished hypotheses: only candidates ranked inside the top num_beams may finish (the rest are spares)
        just_finished = hits & top_k_mask
        gen_now = cur_len + 1 - prompt_len
        fin_scores = cand_scores / (norm_len(gen_now) ** length_penalty)
        if early_stopping is True:
            fin_scores = fin_scores + torch.all(is_finished, dim=-1, keepdim=True).float() * NEG
        fin_scores = fin_scores + (~heuristic_open).float() * NEG + (~just_finished).float() * NEG
        m_seqs = torch.cat([finished, cand], 1)
        m_scores = torch.cat([finished_scores, fin_scores], 1)
        m_len = torch.cat([finished_len, torch.full((B, K), gen_now, dtype=torch.long, device=dev)], 1)
        m_fin = torch.cat([is_finished, just_finished], 1)
        best = torch.topk(m_scores, k, dim=1)[1]
        finished, finished_scores = _gather_beams(m_seqs, best), _gather_beams(m_scores, best)
        finished_len, is_finished = _gather_beams(m_len, best), _gather_beams(m_fin, best)
        cur_len += 1
        # can the best live beam still beat the worst finished hypothesis?
        gen_live = cur_len - prompt_len
        hyp_len = (max_length - prompt_len) if (early_stopping == "never" and length_penalty > 0.0) else gen_live
        best_live = running_scores[:, :1] / (norm_len(hyp_len) ** length_penalty)
        worst_fin = torch.where(is_finished, finished_scores.min(dim=1, keepdim=True)[0], torch.full_like(finished_scores, NEG))
        heuristic_open = heuristic_open & torch.any(best_live > worst_fin, dim=-1, keepdim=True)
        more = bool(torch.any(heuristic_open)) and not (bool(torch.all(is_finished)) and early_stopping is True) and not bool(torch.all(hits))
        if not more:
            break
        cache.reorder((next_src + torch.arange(B, device=dev)[:, None] * k).reshape(-1))
        if graph is not None:
            graph.ids.copy_(running[:, :, cur_len - 1].reshape(B * k))
            logits = graph.replay()
            continue
        if am is not None:                                               # (rows of one sample share a mask: re-ordering beams keeps it)
            am = torch.cat([am, torch.ones_like(am[:, :1])], 1)
            mask_kw = dict(attention_mask=am, position_ids=am.long().sum(-1, keepdim=True) - 1)
        out = model(input_ids=running[:, :, cur_len - 1].reshape(B * k, 1), past_key_values=cache, use_cache=True, last_token_logits_only=True,
                    **mask_kw)
        logits = out.logits[:, -1].float()
    out_len = prompt_len + int(finished_len[:, 0].max())
    seqs = finished[:, 0, :out_len]
    return (seqs, finished_scores[:, 0]) if return_scores else seqs

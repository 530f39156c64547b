"""Per-token decode time of the eager kv-cache step and of the captured `DecodeGraph` step, at the Vicuna-7B shape with random bf16
weights, and `attn_decode` against `attn_fwd_cache` alone (DESIGN.md §4).

    python scripts/decode.py [--layers 32] [--tokens 32] [--rounds 7] [--prompts 512 2048] [--batches 1 5 8 32]

Eager and graph rounds alternate on the same cache (rewound to the prompt between rounds); CUDA events time each round of `--tokens`
steps, and the median and range over `--rounds` rounds of each are printed.  The HBM bound per token is (weight bytes + K/V bytes read)
/ 3.35 TB/s (H100 SXM data sheet).  The GEMM line is the eager step's M = B GEMMs, timed with CUDA events around each launch in a
separate step.  Prints one JSON object per measurement."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def attention_alone(ops, iters=200):
    BF = torch.bfloat16
    nh, d, L = 32, 128, 2048
    for B in (1, 8):
        for nkv in (32, 8):
            g = torch.Generator(device="cuda").manual_seed(0)
            q = torch.randn(B, 1, nh, d, device="cuda", generator=g).to(BF)
            K = torch.randn(B, L + 64, nkv, d, device="cuda", generator=g).to(BF)
            V = torch.randn_like(K)
            kvl = torch.tensor([L], dtype=torch.int32, device="cuda")
            ws = torch.empty(ops.attn_decode_workspace_bytes(B, nh, nkv, d, L + 64), dtype=torch.uint8, device="cuda")
            out = torch.empty(B, nh * d, dtype=BF, device="cuda")
            q3 = q.view(B, nh, d)

            def dec():
                ops.attn_decode(q3, K, V, kvl, workspace=ws, out=out)

            def fc():
                ops.attn_fwd_cache(q, K, V, L, causal=True)

            for f in (dec, fc):
                timed(f, 20)
            t = {"attn_decode": [], "attn_fwd_cache": []}
            for _ in range(3):                                            # alternate the two kernels
                t["attn_decode"].append(timed(dec, iters))
                t["attn_fwd_cache"].append(timed(fc, iters))
            kv_bytes = 2 * B * L * nkv * d * 2
            ns, sl = ops.attn_decode_plan(B, nkv, L + 64)
            for k, v in t.items():
                ms = min(v)
                print(json.dumps({"what": "attention", "kernel": k, "B": B, "nh": nh, "nkv": nkv, "d": d, "kv_len": L, "us": round(ms * 1e3, 2),
                                  "TB/s": round(kv_bytes / (ms * 1e-3) / 1e12, 3), "splits": ns if k == "attn_decode" else None,
                                  "split_len": sl if k == "attn_decode" else None}), flush=True)


def per_token(model, ops, cfg, prompt, B, tokens, rounds):
    from dreamllm_b200.decode import DecodeGraph
    V = cfg.vocab_size
    ids = torch.randint(0, V, (B, prompt), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    with torch.no_grad():
        out = model(input_ids=ids, use_cache=True, last_token_logits_only=True)
    cache = out.past_key_values
    nxt = out.logits[:, -1].argmax(-1)
    del out

    def eager_round():
        cache.len = prompt
        tok = nxt[:, None]

        def one():
            nonlocal tok
            with torch.no_grad():
                o = model(input_ids=tok, past_key_values=cache, use_cache=True, last_token_logits_only=True)
            tok = o.logits[:, -1].argmax(-1)[:, None]
        return timed(one, tokens)

    def graph_round():
        cache.len = prompt
        dg = DecodeGraph(model, cache, B)
        dg.ids.copy_(nxt)
        dg.capture()

        def one():
            dg.ids.copy_(dg.replay().argmax(-1))
        t = timed(one, tokens)
        del dg
        return t

    eager_round()                                                          # warm-up (module loading, GEMM plans)
    res = {"eager": [], "graph": []}
    for _ in range(rounds):
        res["eager"].append(eager_round())
        res["graph"].append(graph_round())
    # the M = B GEMMs of one eager step
    cache.len = prompt
    ops.PROFILE.reset(enabled=True)
    with torch.no_grad():
        model(input_ids=nxt[:, None], past_key_values=cache, use_cache=True, last_token_logits_only=True)
    gemm = ops.PROFILE.summary()
    ops.PROFILE.reset()
    H, I, L = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers
    nh = cfg.num_attention_heads
    nkv = getattr(cfg, "num_key_value_heads", nh)
    d = H // nh
    w_bytes = 2 * (L * (H * (nh + 2 * nkv) * d + nh * d * H + 3 * H * I + 2 * H) + 2 * V * H)
    kv_bytes = 2 * 2 * L * B * (prompt + tokens // 2) * nkv * d
    bound = (w_bytes + kv_bytes) / HBM * 1e3
    del cache
    torch.cuda.empty_cache()
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    return {"what": "per_token", "prompt": prompt, "B": B, "layers": L, "eager_ms_median": round(med["eager"], 3),
            "graph_ms_median": round(med["graph"], 3), "eager_ms_range": [round(min(res["eager"]), 3), round(max(res["eager"]), 3)],
            "graph_ms_range": [round(min(res["graph"]), 3), round(max(res["graph"]), 3)],
            "graph_slower_rounds": sum(g >= e for e, g in zip(res["eager"], res["graph"])), "rounds": rounds,
            "hbm_bound_ms": round(bound, 3), "gemm_ms": round(gemm["ms"], 3), "gemm_launches": gemm["n"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--tokens", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7, help="eager / graph rounds, alternated; the median and the range are printed")
    ap.add_argument("--prompts", type=int, nargs="+", default=[512, 2048])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 5, 8, 32])
    ap.add_argument("--skip-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/decode.py measures on a GPU; none is visible")
    from dreamllm_b200 import _lib, ops
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    _lib.build()
    print(json.dumps(card()), flush=True)
    attention_alone(ops)
    if a.skip_model:
        return
    cfg = DreamLLMConfig(vocab_size=32000, hidden_size=4096, intermediate_size=11008, num_hidden_layers=a.layers, num_attention_heads=32,
                         max_position_embeddings=max(a.prompts) + a.tokens + 64)
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = DreamLLMForCausalMLM(cfg)
    model = model.to(torch.bfloat16).eval()
    for prompt in a.prompts:
        for B in a.batches:
            print(json.dumps(per_token(model, ops, cfg, prompt, B, a.tokens, a.rounds)), flush=True)


if __name__ == "__main__":
    main()

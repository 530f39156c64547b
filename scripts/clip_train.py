"""Time the CLIP ViT-L/14 tower frozen (forward) and trainable (forward + backward), next to transformers' CLIPVisionModel in bf16
on the same card, with random bf16 weights (DESIGN.md §4).

    python scripts/clip_train.py [--rounds 7] [--images 4 16] [--res 336 224] [--profile] [--parent PATH] [--out DIR]

The three workloads alternate within each round; CUDA events time each call, and the median and [min, max] over the rounds are
printed.  TFLOP/s use the analytic count of the 23 computed layers (select_layer -2): per token and layer 2 (4 C^2 + 2 C I) + 4 S C,
i.e. 365.3 GFLOP per image forward at 336 px; the backward counts twice the forward.  `--profile` adds a separate torch.profiler run of
one trainable step at 336 px and reports the LayerNorm-affine and quick-GELU kernels' time and HBM rate against 3.35 TB/s (H100 SXM
data sheet).  `--parent PATH` (a checkout of another revision with its library built) computes the frozen ViT-L/14-336 features
there in a subprocess and checks they are bit-identical to this tree's.  Prints one JSON object per measurement."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HBM = 3.35e12
VIT_L = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16, patch_size=14)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    import torch
    return {"card": torch.cuda.get_device_name(0), "name_power_limit_max_sm_clock": q.stdout.strip()}


def flops_fwd(res, layers=23, C=1024, I=4096):
    S = (res // 14) ** 2 + 1
    return layers * S * (2 * (4 * C * C + 2 * C * I) + 4 * S * C)


def towers(res, seed=0):
    import torch
    from dreamllm_b200.clip_vision import CLIPVisionConfigLite, CLIPVisionModel
    from transformers import CLIPVisionConfig
    from transformers import CLIPVisionModel as HF
    torch.manual_seed(seed)
    hf = HF(CLIPVisionConfig(image_size=res, **VIT_L))
    sd = hf.state_dict()
    frozen = CLIPVisionModel(CLIPVisionConfigLite(image_size=res, **VIT_L))
    frozen.load_state_dict(sd)
    frozen = frozen.to(device="cuda", dtype=torch.bfloat16).requires_grad_(False)
    train = CLIPVisionModel(CLIPVisionConfigLite(image_size=res, **VIT_L))
    train.load_state_dict(sd)
    train = train.to(device="cuda", dtype=torch.bfloat16)
    train.vision_model.encoder.layers[-1].requires_grad_(False)      # the plugin's select_layer -2 rule
    train.vision_model.post_layernorm.requires_grad_(False)
    hf = hf.to(device="cuda", dtype=torch.bfloat16)
    return frozen, train, hf


def frozen_features(res=336, n=2):
    import torch
    frozen, _, _ = towers(res)
    img = torch.randn(n, 3, res, res, generator=torch.Generator().manual_seed(5)).to(torch.bfloat16).cuda()
    return frozen.hidden_state(img, -2).cpu()


def measure(res, N, rounds):
    import torch
    frozen, train, hf = towers(res)
    img = torch.randn(N, 3, res, res, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).cuda()
    S = (res // 14) ** 2 + 1
    gfeat = torch.randn(N, S - 1, 1024, generator=torch.Generator().manual_seed(2)).to(torch.bfloat16).cuda()
    hf_params = [p for p in hf.parameters() if p.requires_grad]

    def f_frozen():
        frozen.hidden_state(img, -2)

    def f_train():
        for p in train.parameters():
            p.grad = None
        train.hidden_state(img, -2)[:, 1:].backward(gfeat)

    def f_hf():
        for p in hf_params:
            p.grad = None
        hf(img, output_hidden_states=True).hidden_states[-2][:, 1:].backward(gfeat)

    fns = {"frozen_fwd": f_frozen, "train_fwd_bwd": f_train, "transformers_bf16_fwd_bwd": f_hf}
    for f in fns.values():                       # warm-up: module loads, allocator, library algorithm picks
        f()
        f()
    torch.cuda.synchronize()
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    mem = {}
    for k, f in fns.items():
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        f()
        torch.cuda.synchronize()
        mem[k] = {"max_memory_allocated_GB": round(torch.cuda.max_memory_allocated() / 1e9, 3),
                  "peak_over_start_GB": round((torch.cuda.max_memory_allocated() - base) / 1e9, 3)}
    fl = flops_fwd(res) * N
    out = []
    for k, v in ms.items():
        med = statistics.median(v)
        work = fl if k == "frozen_fwd" else 3 * fl
        out.append({"what": k, "res": res, "images": N, "rounds": rounds, "ms_median": round(med, 3),
                    "ms_min_max": [round(min(v), 3), round(max(v), 3)], "tflops_analytic": round(work / med / 1e9, 1), **mem[k]})
    del frozen, train, hf
    torch.cuda.empty_cache()
    return out


def profile(res=336, N=16):
    import torch
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as prof
    _, train, _ = towers(res)
    img = torch.randn(N, 3, res, res, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).cuda()
    S = (res // 14) ** 2 + 1
    T, C, I = N * S, 1024, 4096
    g = torch.randn(N, S - 1, C).to(torch.bfloat16).cuda()

    def step():
        for p in train.parameters():
            p.grad = None
        train.hidden_state(img, -2)[:, 1:].backward(g)

    step()
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        step()
        torch.cuda.synchronize()
    # bytes each launch must move (bf16 = 2 B): LN affine dx pass reads dy, x, dres and writes dx (+ (mean, rstd) per row); the
    # weight pass reads dy and x again; quick-GELU reads x and writes y; its backward reads dy and x and writes dx
    kinds = {"layernorm_bwd_warp_kernel<4, true>": 4 * T * C * 2 + 8 * T, "layernorm_bwd_dwb_kernel": 2 * T * C * 2 + 8 * T,
             "layernorm_dwb_final_kernel": 64 * 2 * C * 4 + 4 * C, "quick_gelu_kernel": 2 * T * I * 2, "quick_gelu_bwd_kernel": 3 * T * I * 2}
    acc = {}
    for e in p.events():
        if e.device_type is None or "cuda" not in str(e.device_type).lower():
            continue
        name = e.name.replace("dllm::", "").replace("(anonymous namespace)::", "")
        for k in kinds:
            stem = k.split("<")[0]
            if stem in name and (("true" in name) == ("true" in k) if stem == "layernorm_bwd_warp_kernel" else True):
                if stem == "quick_gelu_kernel" and "bwd" in name:
                    continue
                acc.setdefault(k, []).append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
    out = []
    for k, ts in acc.items():
        us = statistics.mean(ts)
        out.append({"what": "kernel", "kernel": k, "res": res, "images": N, "launches": len(ts), "us_mean": round(us, 1),
                    "GB_per_s": round(kinds[k] / us / 1e3, 1), "of_3.35TB_s": round(kinds[k] / (us * 1e-6) / HBM, 3)})
    for k in kinds:
        if k not in acc:
            out.append({"what": "kernel", "kernel": k, "result": "not measured (no matching profiler event)"})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--images", type=int, nargs="+", default=[4, 16])
    ap.add_argument("--res", type=int, nargs="+", default=[336, 224])
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--parent", default="", help="checkout of another revision (library built): frozen features must be bit-identical")
    ap.add_argument("--features-out", default="", help=argparse.SUPPRESS)
    ap.add_argument("--tree", default=ROOT, help=argparse.SUPPRESS)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    sys.path.insert(0, a.tree)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("clip_train.py measures on a GPU; no CUDA device is visible")
    if a.features_out:
        torch.save(frozen_features(), a.features_out)
        return
    lines = [{**card(), "transformers_attention": "sdpa (transformers' default)"}]
    print(json.dumps(lines[0]), flush=True)
    if a.parent:
        with tempfile.TemporaryDirectory() as tmp:
            f = os.path.join(tmp, "parent.pt")
            env = {k: v for k, v in os.environ.items() if k != "DLLM_LIB_PATH"}
            subprocess.run([sys.executable, os.path.abspath(__file__), "--features-out", f, "--tree", os.path.abspath(a.parent)],
                           cwd=a.parent, check=True, env=env)
            theirs = torch.load(f)
        ours = frozen_features()
        rec = {"what": "frozen ViT-L/14-336 features vs parent", "bit_identical": bool(torch.equal(ours, theirs)),
               "max_abs_diff": float((ours.float() - theirs.float()).abs().max())}
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    for res in a.res:
        for N in a.images:
            for rec in measure(res, N, a.rounds):
                lines.append(rec)
                print(json.dumps(rec), flush=True)
    if a.profile:
        for rec in profile():
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "clip_train.jsonl"), "w") as fh:
            fh.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()

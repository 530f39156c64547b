"""Where the headline step's GEMM time goes, and what each N-tile width costs (dev tool, needs one H100).

  python scripts/gemm_shapes.py profile     one eager c5 step (bench.py's stage-1 step) with ops.PROFILE on: launches, time and TFLOP/s
                                            per (M, N, K, mode) group, largest time first
  python scripts/gemm_shapes.py widths      the fixed c5 shape table below, timed with CUDA events over many launches, once per N-tile
                                            width (DLLM_GEMM_BN pins the width; one child process per width) and once as planned
  python scripts/gemm_shapes.py tilecost    the same table plus two VAE-encoder convolutions and one split-K linear, each timed at K and at
                                            2K (same M, N and width): fixed = 2 t(K) - t(2K) is the part of the launch that does not scale
                                            with K (tile prologue + epilogue), printed per wave of tiles next to t(K)
  python scripts/gemm_shapes.py all         profile and widths

Runs on whichever library DLLM_LIB_PATH names (default: the in-tree build), so two builds can be compared side by side.  A build older
than the tile planner ignores DLLM_GEMM_BN and has no dllm_gemm_tile_n; its rows then all show its own fixed widths.
"""
from __future__ import annotations

import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from dreamllm_b200 import _lib  # noqa: E402


def _load():
    """Drop ctypes signatures the library under test does not export (builds that predate them), then load it."""
    import ctypes
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for name in list(_lib.SIGNATURES):
        if not hasattr(raw, name):
            del _lib.SIGNATURES[name]
    return _lib.lib()


# (kind, M, N, K) of the stage-1 step's unsplit launches with K-major A; conv rows are (N images, H = W, Cin, Cout) as M = N*H*W,
# N = Cout, K = 9*Cin.  UNet on 4 samples at 64x64 / 32x32 latents, the 7B LLM on 400 tokens.
SHAPES = [
    ("fwd", 16384, 320, 320), ("fwd", 16384, 320, 1280), ("fwd", 16384, 960, 320), ("fwd", 16384, 2560, 320),
    ("fwd", 4096, 640, 640), ("fwd", 4096, 640, 2560), ("fwd", 4096, 1920, 640),
    ("fwd", 400, 12288, 4096), ("fwd", 400, 22016, 4096),
    ("dgrad", 16384, 320, 320), ("dgrad", 16384, 320, 1280), ("dgrad", 16384, 320, 960), ("dgrad", 4096, 640, 640),
    ("dgrad", 4096, 640, 2560), ("dgrad", 400, 11008, 4096),
    ("conv", 16384, 320, 9 * 320), ("conv", 16384, 320, 9 * 640), ("conv", 4096, 640, 9 * 640), ("conv", 4096, 640, 9 * 1280),
]
WIDTHS = (256, 224, 192, 160, 128)
# tilecost only: VAE encoder 3x3 convolutions at the full- and half-resolution levels of 4 images of 512x512, and the UNet's 16x16-level
# linear (a split-K launch: its fixed part includes the fp32 partial store and the reduce kernel)
TILECOST_EXTRA = [("conv", 4 * 512 * 512, 128, 9 * 128), ("conv", 4 * 256 * 256, 256, 9 * 256), ("fwd", 1024, 1280, 1280)]


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _bench_one(kind, M, N, K):
    from dreamllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    if kind == "conv":
        side = int(round((M // 4) ** 0.5))
        cin = K // 9
        x = torch.randn(4, side, side, cin, device="cuda", generator=g).to(torch.bfloat16)
        w = (torch.randn(N, K, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        bias = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
        fn = lambda: ops.conv3x3(x, w, bias=bias)   # noqa: E731
    else:
        a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
        b = (torch.randn((K, N) if kind == "dgrad" else (N, K), device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        fn = lambda: ops.gemm(a, b, b_mn=(kind == "dgrad"), out=out)   # noqa: E731
    flop = 2.0 * M * N * K
    iters = max(20, min(2000, int(2e13 / flop)))     # ~ 20 ms of work per timing
    return min(_time(fn, iters) for _ in range(3))


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def tilecost():
    L = _load()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"\ncard: {_card()}; {sms} SMs")
    print("fixed = 2 t(K) - t(2K): the time of a launch that does not scale with K; per wave = fixed / ceil(tiles / SMs)")
    print(f"{'kind':6s} {'M':>8s} {'N':>6s} {'K':>6s} {'bn':>4s} {'waves':>5s} | {'t(K) us':>9s} {'t(2K) us':>9s} | {'fixed us':>9s} "
          f"{'per wave':>9s} {'of t(K)':>8s}")
    for kind, M, N, K in SHAPES + TILECOST_EXTRA:
        b_mn = int(kind == "dgrad")
        bn = L.dllm_gemm_tile_n(M, N, K, b_mn)
        if L.dllm_gemm_tile_n(M, N, 2 * K, b_mn) != bn:
            raise RuntimeError(f"{(kind, M, N, K)}: K and 2K plan different widths")
        split = "*" if M <= 4096 and L.dllm_gemm_splitk_workspace_bytes(M, N, K) else " "
        t1 = _bench_one(kind, M, N, K) * 1e3
        t2 = _bench_one(kind, M, N, 2 * K) * 1e3
        waves = -(-((M + 127) // 128 * -(-N // bn)) // sms)
        fixed = 2 * t1 - t2
        print(f"{kind:6s} {M:8d} {N:6d} {K:6d} {bn:4d} {waves:5d} | {t1:9.1f} {t2:9.1f} | {fixed:9.1f} {fixed / waves:9.2f} "
              f"{100 * fixed / t1:7.1f}%{split}")
    print("* split-K launch (fp32 partials + reduce kernel)")


def widths_child():
    """One process = one pinned width (the library reads DLLM_GEMM_BN once)."""
    L = _load()
    rows = []
    for kind, M, N, K in SHAPES:
        bn = L.dllm_gemm_tile_n(M, N, K, int(kind == "dgrad")) if hasattr(L, "dllm_gemm_tile_n") else None
        rows.append({"kind": kind, "M": M, "N": N, "K": K, "bn": bn, "ms": _bench_one(kind, M, N, K)})
    print(json.dumps(rows))


def widths():
    res = {}
    pinned = WIDTHS if hasattr(_load(), "dllm_gemm_tile_n") else ()
    for w in ("planned",) + pinned:
        env = dict(os.environ)
        env.pop("DLLM_GEMM_BN", None)
        if w != "planned":
            env["DLLM_GEMM_BN"] = str(w)
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "_widths_child"], env=env, capture_output=True, text=True, check=True)
        res[w] = json.loads(out.stdout.strip().splitlines()[-1])
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"\nper-shape time (us) by N-tile width; 'planned' = the library's own choice (its width in brackets); {sms} SMs")
    print(f"{'kind':6s} {'M':>6s} {'N':>6s} {'K':>6s} | {'planned':>14s} | " + " | ".join(f"{w:>8d}" for w in pinned))
    ratios = {w: [] for w in pinned}
    for i, (kind, M, N, K) in enumerate(SHAPES):
        p = res["planned"][i]
        cells = []
        for w in pinned:
            r = res[w][i]
            ok = r["bn"] == w or r["bn"] is None
            cells.append(f"{r['ms'] * 1e3:8.1f}" if ok else f"{'-':>8s}")
            # per-wave time relative to 256 on the many-wave shapes: the planner's t(width)
            tiles = (M + 127) // 128 * -(-N // w)
            if ok and r["bn"] == w and M >= 4096 and res[256][i]["bn"] == 256:
                waves, waves256 = -(-tiles // sms), -(-((M + 127) // 128 * -(-N // 256)) // sms)
                ratios[w].append((r["ms"] / waves) / (res[256][i]["ms"] / waves256))
        print(f"{kind:6s} {M:6d} {N:6d} {K:6d} | {p['ms'] * 1e3:8.1f} [{p['bn']}] | " + " | ".join(cells))
    print("\nper-wave time relative to 256 (M >= 4096 rows): median [min, max]")
    for w in pinned:
        v = ratios[w]
        if v:
            print(f"  {w}: {statistics.median(v):.3f} [{min(v):.3f}, {max(v):.3f}] over {len(v)} shapes")


def profile():
    """One eager stage-1 step in steady state: bench.run_c5 with the CUDA graph off, PROFILE on for its first timed step only."""
    import argparse

    import bench
    from dreamllm_b200 import ops

    class ProfEnv(bench.Env):
        groups = None

        def timed(self, fn, k):
            if self.groups is not None:
                return super().timed(fn, k)
            ops.PROFILE.reset(enabled=True)
            t = super().timed(fn, k)
            self.groups = ops.PROFILE.by_shape()
            ops.PROFILE.reset(enabled=False)
            return t

    os.environ["DLLM_STAGE1_GRAPH"] = "0"
    env = ProfEnv(argparse.Namespace())
    model = bench.build_llm(env, bench.L)
    step_ms = bench.run_c5(env, model, 1, 2)["ms_per_step"]
    rows = sorted(env.groups.items(), key=lambda kv: -kv[1][1])
    tot_ms = sum(r[1] for _, r in rows)
    tot_fl = sum(r[2] for _, r in rows)
    print(f"\none eager c5 step: {step_ms:.1f} ms; GEMM + conv launches {tot_ms:.1f} ms ({len(rows)} shapes, "
          f"{sum(r[0] for _, r in rows)} launches, {tot_fl / 1e12:.2f} TFLOP, {tot_fl / 1e9 / tot_ms:.0f} TFLOP/s)")
    print(f"{'mode':8s} {'M':>6s} {'N':>6s} {'K':>6s} {'n':>4s} {'ms':>8s} {'share':>6s} {'TFLOP/s':>8s}")
    for (M, N, K, mode), (n, ms, fl) in rows:
        print(f"{mode:8s} {M:6d} {N:6d} {K:6d} {n:4d} {ms:8.3f} {100 * ms / tot_ms:5.1f}% {fl / 1e9 / ms:8.0f}")


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    if what == "_widths_child":
        widths_child()
        sys.exit(0)
    if not torch.cuda.is_available():
        raise RuntimeError("gemm_shapes.py needs a CUDA device")
    _load()
    print(f"library: {_lib.LIB_PATH}")
    if what in ("profile", "all"):
        profile()
    if what in ("widths", "all"):
        widths()
    if what == "tilecost":
        tilecost()

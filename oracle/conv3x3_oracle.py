"""TEST INFRASTRUCTURE ONLY — float64 references for the implicit-GEMM 3x3 convolution (`dllm_conv3x3_nhwc[_ws]`, `ops.conv3x3`).

Plain torch on the host (no `dreamllm_b200` import).  The kernel computes every output as one fp32 accumulation of bf16 x bf16
products and rounds where its epilogue rounds; the reference does the sum in float64 and rounds at the same points.  The geometry
table, the seeded inputs and the comparison used by tests/test_conv3x3_gpu.py live here too, so that tests/test_conv3x3_cpu.py can show
on the very same inputs that the comparison rejects a kernel that is subtly wrong.

The conv's A tile is a 4-D TMA box {64 c, Wb, Hb, Nb} of 128 pixels (csrc/gemm_sm90.cu, conv3x3_nhwc_ws):
    int Wb = W > 128 ? 128 : W, Hb = W > 128 ? 1 : 128 / W, Nb = 1;
    if (Hb > H) { ... Nb = Hb / H; Hb = H; }
so the plane's W picks one of four tile shapes (`box_class`): part of one row ("seam", W > 128: the tile origin has w0 != 0), exactly
one row ("row", W == 128), several rows of one image ("rows") and several whole images ("images", the last tile may hang past the
batch).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn.functional as F

BF = torch.bfloat16
F64 = torch.float64

# Per-element fp32 accumulation slack of the kernel, as a fraction of term_mass (sum over the K terms of |x| |w|).  The largest
# needed on an H100 80GB HBM3 (700 W) over every case of CASES and DGRAD_CASES was 4.1e-7 (K = 9 x 1280, unsplit); 2^-20 = 9.5e-7
# leaves 2x.  tests/test_conv3x3_cpu.py requires it to stay 10x below the smallest injected fault signal (1.9e-2, a dropped tap).
C_ACC = 2.0 ** -20


def bf16r(x: torch.Tensor) -> torch.Tensor:
    """Round to bf16 (round to nearest even) and back to float64."""
    return x.to(torch.float32).to(BF).to(F64)


def ulp(v: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 at |v| (v a float64 tensor of bf16 values): 2^(e - 7) for |v| in [2^e, 2^(e+1))."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def box_plan(H: int, W: int):
    """(Wb, Hb, Nb) of the A tile, or None where conv3x3_nhwc_ws refuses the plane."""
    if H <= 0 or W <= 0 or (W % 128 if W > 128 else 128 % W):
        return None
    if W > 128:
        return 128, 1, 1
    hb = 128 // W
    if hb > H:
        return (W, H, hb // H) if hb % H == 0 else None
    return (W, hb, 1) if H % hb == 0 else None


def box_class(H: int, W: int) -> str:
    wb, hb, nb = box_plan(H, W)
    if W > 128:
        return "seam"
    if W == 128:
        return "row"
    return "rows" if nb == 1 else "images"


# ------------------------------------------------------------------------------------------------ references
def _w4(w_k: torch.Tensor) -> torch.Tensor:
    """[Cout, 9 * Cin] with k = (r, s, c) (ops.conv3x3_weight) -> Conv2d weight [Cout, Cin, 3, 3] in float64."""
    Cout = w_k.shape[0]
    return w_k.to(F64).reshape(Cout, 3, 3, -1).permute(0, 3, 1, 2)


def conv3x3_acc(x_nhwc: torch.Tensor, w_k: torch.Tensor) -> torch.Tensor:
    """The accumulator: float64 conv2d(padding=1) of the bf16 values, NHWC."""
    return F.conv2d(x_nhwc.to(F64).permute(0, 3, 1, 2), _w4(w_k), padding=1).permute(0, 2, 3, 1)


def epilogue_ref(acc, bias=None, rowbias=None, residual=None):
    """(t, y, pre): the kernel's epilogue on a float64 accumulator [N, H, W, Cout].  epi_apply (gemm_sm90.cu) does
        x0 += bb.x; ... if (has_rb) { x0 += rb.x; ... }              bias and rowbias[row / rows_per_group] (rows_per_group = HW)
        if (has_rs) { x0 = bf16_round(x0) + rs.x; ... }              rounded, then the residual added
    and the store rounds once more (pack_bf16); splitk_reduce_kernel adds the same operands in the same order.  t is the value before
    the residual add (None without a residual), y the bf16 result and pre the value y is the rounding of."""
    pre = acc
    if bias is not None:
        pre = pre + bias.to(F64)
    if rowbias is not None:
        pre = pre + rowbias.to(F64)[:, None, None, :]
    if residual is None:
        return None, bf16r(pre), pre
    t = bf16r(pre)
    pre = t + residual.to(F64)
    return t, bf16r(pre), pre


def conv3x3_ref(x_nhwc, w_k, bias=None, rowbias=None, residual=None):
    """y[n, h, w, :] = bf16(bf16(conv3x3(x, w) + bias + rowbias[n]) + residual), float64 values of the bf16 result."""
    return epilogue_ref(conv3x3_acc(x_nhwc, w_k), bias, rowbias, residual)[1]


def conv3x3_dgrad_ref(dy_nhwc: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """dx of y = conv2d(x, weight, padding=1): conv2d_input in float64, NHWC (weight [Cout, Cin, 3, 3])."""
    N, H, W, _ = dy_nhwc.shape
    dx = torch.nn.grad.conv2d_input((N, weight.shape[1], H, W), weight.to(F64), dy_nhwc.to(F64).permute(0, 3, 1, 2), padding=1)
    return dx.permute(0, 2, 3, 1)


def term_mass(x_nhwc: torch.Tensor, w_k: torch.Tensor) -> torch.Tensor:
    """Sum over the K terms of |x| |w| for every output element: conv2d(|x|, |w|) in float64.  An fp32 accumulation of those terms is
    off by at most a small multiple of 2^-24 times this."""
    return conv3x3_acc(x_nhwc.abs(), w_k.abs())


# ------------------------------------------------------------------------------------------------ the comparison
def allowance(t, y, mass, c=C_ACC):
    """Per-element bound on |got - y|: one bf16 ulp at every rounding point the value passes (the result, and the pre-residual value
    when a residual follows) plus c x term_mass for the fp32 accumulation."""
    a = ulp(y) + c * mass
    return a if t is None else a + ulp(t)


def slack_needed(got, t, y, mass):
    """Smallest c with |got - y| <= allowance(t, y, mass, c) everywhere (0 when the rounding points alone explain the difference)."""
    excess = (got.to(F64) - y).abs() - allowance(t, y, mass, 0.0)
    return float((excess / mass.clamp_min(1e-300)).clamp_min(0.0).max())


def check_conv(got, t, y, mass, pre, c=C_ACC, max_frac=1e-2, what=""):
    """Raise AssertionError unless every element is within allowance(t, y, mass, c) of y, and at most `max_frac` of the elements whose
    rounding the slack cannot flip differ from y at all.  `got` is the kernel's bf16 output (any device), t / y / pre / mass come from
    epilogue_ref / term_mass.  An element whose unrounded value `pre` lies within c x term_mass (plus an ulp of t, which may itself
    have rounded the other way) of a bf16 rounding midpoint may round to either neighbour: at K = 9 x 2560 over 1 % of N(0, 1) outputs
    are that close to zero, where the ulp is finest."""
    got = got.cpu().to(F64)
    err = (got - y).abs()
    bad = err > allowance(t, y, mass, c)
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), y.shape))
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside one ulp + c * term_mass (c = {c:.3g}); first "
                             f"at [n, h, w, c] = {idx}: got {float(got.flatten()[i])}, reference {float(y.flatten()[i])}")
    near = ulp(y) / 2 - (pre - y).abs() <= c * mass + (0.0 if t is None else ulp(t))
    frac = float(((err > 0) & ~near).double().mean())
    assert frac <= max_frac, f"{what}: {frac:.4f} of the elements differ from the reference (at most {max_frac} allowed)"


# ------------------------------------------------------------------------------------------------ geometries and inputs
@dataclass(frozen=True)
class Case:
    N: int
    H: int
    W: int
    Cin: int
    Cout: int
    split: bool     # ops.conv3x3 takes split-K (N H W <= 4096 and the planner splits, 132 SMs)

    @property
    def id(self) -> str:
        return f"{box_class(self.H, self.W)}-w{self.W}-{self.N}x{self.H}x{self.W}-{self.Cin}to{self.Cout}"


# W covers 512 / 256 / 128 / 64 / 32 / 16 / 8 / 4; every class has planes with H < W and H > W; cpt = Cin / 64 in {1, 2, 5, 20, 40};
# Cout 328 leaves a tail on the N tile.  The "images" planes put 2, 4 or 8 whole images into a tile and leave the last tile partial.
CASES = [
    Case(1, 3, 512, 128, 128, True),      # VAE 512² level: four tiles to a row, seams at w = 128, 256, 384
    Case(1, 260, 256, 64, 8, False),      # VAE 256²-wide plane, H > W
    Case(2, 1, 256, 320, 328, True),      # one-row images: every tap of rows r = 0, 2 is padding; an image boundary at a tile boundary
    Case(1, 6, 128, 320, 320, True),      # SDXL level 0 (C 320)
    Case(1, 132, 128, 64, 8, False),      # one row per tile, H > W
    Case(2, 16, 64, 128, 320, True),      # SD-2.1 / SDXL 64 level: two rows per tile, H < W
    Case(3, 64, 32, 64, 128, False),      # four rows per tile, H > W
    Case(1, 8, 32, 1280, 320, True),
    Case(1, 8, 16, 2560, 128, True),      # SD-2.1 up-block concatenation (cpt 40); one 8 x 16 image per tile
    Case(3, 16, 16, 64, 1280, True),      # SD-2.1 16 level
    Case(1, 16, 8, 128, 320, True),       # W = 8 with Hb = H: one image per tile, H > W
    Case(1, 8, 8, 1280, 320, True),       # SD-2.1 8 level: two images per tile, the only tile half empty
    Case(3, 8, 8, 320, 328, True),        # two images per tile, last tile half empty
    Case(67, 8, 8, 128, 128, False),      # two images per tile, 34 tiles, the last half empty; too many pixels for split-K
    Case(5, 4, 8, 64, 8, True),           # 4 x 8 planes, four images per tile, last tile one image
    Case(3, 8, 4, 128, 128, True),        # 8 x 4 planes, four images per tile, last tile three
    Case(3, 4, 4, 2560, 8, True),         # 4 x 4 planes, eight images per tile, the only tile three eighths full
]

# Frozen-UNet dgrad convs: dx = conv3x3(dy, conv3x3_dgrad_weight(w)).  (N, H, W, Cin, Cout) of the FORWARD conv: SD-2.1's 64 / 32 / 16 /
# 8 levels and SDXL's 128 level with fewer rows and samples.
DGRAD_CASES = [(1, 8, 64, 320, 320), (1, 8, 32, 640, 640), (1, 4, 16, 1280, 1280), (1, 8, 8, 1280, 1280), (1, 2, 128, 320, 320)]


def _g(seed):
    return torch.Generator().manual_seed(seed)


def conv_inputs(case: Case, seed: int = 0):
    """Seeded host inputs of one case: x [N, H, W, Cin], w_k [Cout, 9 Cin], bias [Cout], rowbias [N, Cout], residual [N, H, W, Cout],
    all bf16 with outputs of order one."""
    N, H, W, Cin, Cout = case.N, case.H, case.W, case.Cin, case.Cout
    s = seed + 7919 * (N + 3 * H + 5 * W + 11 * Cin + 13 * Cout)
    x = torch.randn(N, H, W, Cin, generator=_g(s)).to(BF)
    w_k = (torch.randn(Cout, 9 * Cin, generator=_g(s + 1)) / (9 * Cin) ** 0.5).to(BF)
    bias = (0.5 * torch.randn(Cout, generator=_g(s + 2))).to(BF)
    rowbias = (0.5 * torch.randn(N, Cout, generator=_g(s + 3))).to(BF)
    residual = torch.randn(N, H, W, Cout, generator=_g(s + 4)).to(BF)
    return x, w_k, bias, rowbias, residual


EPILOGUES = ("plain", "bias_rowbias", "bias_residual")


def epilogue_operands(epi, bias, rowbias, residual):
    """(bias, rowbias, residual) of one epilogue variant: none; bias + rowbias (ResnetBlock2D.conv1 with the time embedding); bias +
    residual (conv2 with the shortcut)."""
    return {"plain": (None, None, None), "bias_rowbias": (bias, rowbias, None), "bias_residual": (bias, None, residual)}[epi]

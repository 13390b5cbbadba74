"""Reference arithmetic of the FP8 (e4m3) MLP contract (include/osb200.h, osb_gemm_fp8), for the tests.

- `e4m3_round`: round-to-nearest-even onto the grid of finite e4m3 values, saturating at +-448.  It is built from the
  grid itself (every finite e4m3 magnitude), not from torch's float8 cast, so it checks that cast as well.
- `quantize` / `dequantize`: per-row scale s = amax(|row|) / 448 (1 for an all-zero row), codes e4m3(row / s).
- `emulated_mlp` / `fp8_mlps`: the oracle's block MLP in fp32 arithmetic on dequantized operands, rounded where the
  product rounds: fc1's input is the fp32 LN+modulate value, fc2's input is the GELU output rounded to bf16, and the
  weights are quantized per output channel."""
import contextlib

import torch
import torch.nn.functional as F

E4M3_MAX = 448.0
# every finite non-negative e4m3 value, ascending (bit patterns 0x00..0x7e; 0x7f is NaN)
_GRID = torch.arange(0, 0x7F, dtype=torch.uint8).view(torch.float8_e4m3fn).double()


def e4m3_round(x: torch.Tensor) -> torch.Tensor:
    """x (any float dtype) -> the nearest e4m3 value (ties to the even code), saturated to +-448, as float64."""
    grid = _GRID.to(x.device)
    a = x.double().abs().clamp(max=E4M3_MAX)
    hi = torch.searchsorted(grid, a).clamp(max=grid.numel() - 1)     # first grid value >= a
    lo = (hi - 1).clamp(min=0)
    d_lo, d_hi = a - grid[lo], grid[hi] - a
    pick_hi = (d_hi < d_lo) | ((d_hi == d_lo) & (hi % 2 == 0))        # code index parity = mantissa LSB
    return torch.where(pick_hi, grid[hi], grid[lo]) * torch.sign(x.double())


def row_scale(x: torch.Tensor) -> torch.Tensor:
    amax = x.float().abs().amax(-1)
    return torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))


def quantize(x: torch.Tensor):
    """fp32 rows [.., K] -> (codes as float64 e4m3 values, fp32 scales [..])."""
    s = row_scale(x)
    return e4m3_round(x.float() / s[..., None]), s


def dequantize(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    return (q * s[..., None].double()).float()


def qdq(x: torch.Tensor) -> torch.Tensor:
    return dequantize(*quantize(x))


def emulated_mlp(mlp, x: torch.Tensor) -> torch.Tensor:
    """oracle Mlp (fc1 -> GELU-tanh -> fc2) at the FP8 rounding points, fp32 arithmetic; x is the LN+modulate output
    [.., C] of the oracle (fp32, or bf16 when the oracle runs in bf16), the result comes back in x's dtype."""
    shape = x.shape
    xf = x.reshape(-1, shape[-1]).float()
    h = F.gelu(qdq(xf) @ qdq(mlp.fc1.weight).t() + mlp.fc1.bias.float(), approximate="tanh")
    h = h.to(torch.bfloat16).float()
    y = qdq(h) @ qdq(mlp.fc2.weight).t() + mlp.fc2.bias.float()
    return y.reshape(*shape[:-1], -1).to(x.dtype)


@contextlib.contextmanager
def fp8_mlps(oracle):
    """Run every block MLP (spatial and temporal) of the oracle STDiT3 through `emulated_mlp` inside the block; the
    caption MLP keeps its arithmetic, as the product's does.  With the oracle in bf16 this is the FP8 product's rounding
    model: bf16 where the reference's own bf16 path rounds, e4m3 at the MLP operands."""
    blocks = [b for pair in zip(oracle.spatial_blocks, oracle.temporal_blocks) for b in pair]
    for b in blocks:
        b.mlp.forward = (lambda m: (lambda x: emulated_mlp(m, x)))(b.mlp)
    try:
        yield oracle
    finally:
        for b in blocks:
            del b.mlp.forward


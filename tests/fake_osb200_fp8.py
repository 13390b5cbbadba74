"""FP8 entries of the CPU stand-in of the `osb200` binding (TEST INFRASTRUCTURE, not a fallback): torch restatements of
`gemm_fp8`, `ln_modulate_fp8` and `quant_rows_fp8` (include/osb200.h) with the kernels' refusals and the launch-count
convention of tests/fake_osb200.py.  Quantization follows the contract: s = amax(|row|) / 448 (1 for a zero row), codes
= the torch float8_e4m3fn cast of row / s (round to nearest even; |row / s| <= 448 by construction, the clamp only states
the kernels' satfinite).  The GEMM sums the e4m3 products in fp32 and applies acc * (a_scale * w_scale) + bias before the
epilogue, with one rounding to bf16.

`install(monkeypatch)` adds these entries to tests/fake_osb200.py for the duration of one test, the way
tests/fake_osb200_text.py adds the text-encoder entries."""
import torch
import torch.nn.functional as F

from tests import fake_osb200 as base

OsbError = base.OsbError
E4M3 = torch.float8_e4m3fn


def install(monkeypatch) -> None:
    for name in ("gemm_fp8", "ln_modulate_fp8", "quant_rows_fp8"):
        monkeypatch.setattr(base, name, globals()[name], raising=False)


def _quant(x):
    """fp32 rows -> (e4m3 codes, fp32 scales)."""
    amax = x.abs().amax(-1)
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (x / s[:, None]).clamp(-448.0, 448.0).to(E4M3), s


def _put(val, out):
    if out is None:
        return val
    out.copy_(val)
    return out


def quant_rows_fp8(x, *, out=None, out_scale=None):
    base._need(x, torch.bfloat16, "x")
    if x.dim() != 2:
        raise OsbError(f"quant_rows_fp8: x must be [rows, K], got {tuple(x.shape)}")
    rows, K = x.shape
    if K % 8 or K > 8192:
        raise OsbError(f"osb_quant_rows_fp8 failed (-1): K must be a multiple of 8 and <= 8192 (got {K})")
    if x.stride(0) % 8:
        raise OsbError("osb_quant_rows_fp8 failed (-1): ldx must be a multiple of 8")
    q, s = _quant(x.float())
    base._count("quant_rows_fp8", (rows, K))
    return _put(q, out), _put(s, out_scale)


def ln_modulate_fp8(x, shift, scale, *, group_rows: int, mod_index=None, eps: float = 1e-6, out=None, out_scale=None):
    base._need(x, torch.bfloat16, "x"); base._need(shift, torch.float32, "shift"); base._need(scale, torch.float32, "scale")
    base._need(mod_index, torch.int32, "mod_index")
    assert x.dim() == 2 and x.is_contiguous()
    assert shift.dim() == 2 and scale.dim() == 2 and shift.stride(0) == scale.stride(0)
    rows, C = x.shape
    if C % 8 or C > 4096:
        raise OsbError(f"osb_ln_modulate_fp8 failed (-1): C must be a multiple of 8 and <= 4096 (got {C})")
    xf = x.float()
    mu = xf.mean(-1, keepdim=True)
    var = (xf - mu).pow(2).mean(-1, keepdim=True)
    g = base._groups(rows, group_rows, mod_index, x.device)
    y = (xf - mu) * torch.rsqrt(var + eps) * (1.0 + scale[g]) + shift[g]   # fp32, not rounded to bf16
    q, s = _quant(y)
    base._count("ln_modulate_fp8", (rows, C))
    return _put(q, out), _put(s, out_scale)


def gemm_fp8(a8, a_scale, w8, w_scale, bias=None, *, epilogue: int = base.EPI_BIAS, residual=None, gate=None,
             group_rows: int = 0, mod_index=None, out=None, block_n: int = 0):
    base._need(a8, E4M3, "a8"); base._need(w8, E4M3, "w8")
    base._need(a_scale, torch.float32, "a_scale"); base._need(w_scale, torch.float32, "w_scale")
    for t, n in ((bias, "bias"), (residual, "residual"), (out, "out")):
        base._need(t, torch.bfloat16, n)
    base._need(gate, torch.float32, "gate"); base._need(mod_index, torch.int32, "mod_index")
    if a8.dim() != 2 or w8.dim() != 2 or a8.shape[1] != w8.shape[1]:
        raise OsbError(f"gemm_fp8: a8 [M, K] and w8 [N, K] expected, got {tuple(a8.shape)} and {tuple(w8.shape)}")
    M, K = a8.shape
    N = w8.shape[0]
    if a_scale is None or w_scale is None or a_scale.shape != (M,) or w_scale.shape != (N,):
        raise OsbError(f"gemm_fp8: a_scale must be [{M}] and w_scale [{N}]")
    base._epilogue_shapes("gemm_fp8", M, N, N, out, bias, residual, gate, group_rows, mod_index)
    if K % 128:
        raise OsbError(f"osb_gemm_fp8 failed (-1): osb_gemm_fp8: K must be a multiple of 128 (one e4m3 k-block), got {K}")
    if N % 8:
        raise OsbError(f"osb_gemm_fp8 failed (-1): osb_gemm_fp8: N must be a multiple of 8, got {N}")
    if block_n not in (0, 64, 128):
        raise OsbError(f"osb_gemm_fp8 failed (-3): osb_gemm_fp8: unsupported block_n {block_n} (64 or 128)")
    if not base.EPI_BIAS <= epilogue <= base.EPI_BIAS_GATE_RES:
        raise OsbError(f"osb_gemm_fp8 failed (-1): osb_gemm_fp8: epilogue {epilogue} is not built for FP8")
    acc = (a8.float() @ w8.float().t()) * (a_scale[:, None] * w_scale[None, :])
    if bias is not None:
        acc = acc + bias.float()
    if epilogue == base.EPI_BIAS_GELU_TANH:
        acc = F.gelu(acc, approximate="tanh")
    elif epilogue == base.EPI_BIAS_GATE_RES:
        if gate is not None:
            acc = acc * gate[base._groups(M, group_rows if group_rows > 0 else M, mod_index, a8.device)]
        if residual is not None:
            acc = acc + residual.float()
    base._count("gemm_fp8", (M, N, K, epilogue))
    return _put(acc.to(torch.bfloat16), out)

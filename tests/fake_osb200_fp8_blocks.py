"""Block-scaled FP8 entries of the CPU stand-in of the `osb200` binding (TEST INFRASTRUCTURE, not a fallback): torch
restatements of `gemm_fp8_blocks` and `quant_blocks_fp8` (include/osb200.h, osb_gemm_fp8_blocks / osb_quant_blocks_fp8)
with the kernels' refusals and the launch-count convention of tests/fake_osb200.py, layered on tests/fake_osb200_fp8.py.

- Block rule: the block (r, b) = X[r, 128 b : 128 b + 128] gets s = amax / 448 (1 for a zero block), codes = the torch
  float8_e4m3fn cast of X / s (round to nearest even).  `block = K` is the per-row rule over rows of any length.
- The GEMM sums each 128-element k-block's e4m3 products, multiplies the partial by a_scale[m, kb] and adds it into the
  accumulator (in `fake_osb200.ACC_DTYPE`), then applies w_scale[n], the bias and the epilogue.  The FP8 GELU epilogue
  quantizes the fp32 GELU value per (row, 128 columns) with the block rule.

`install(monkeypatch)` adds these entries (and those of tests/fake_osb200_fp8.py) to tests/fake_osb200.py for one test."""
import torch
import torch.nn.functional as F

from tests import fake_osb200 as base
from tests import fake_osb200_fp8 as f8

OsbError = base.OsbError
E4M3 = torch.float8_e4m3fn
EPI_BIAS_GELU_TANH_FP8 = 5


def install(monkeypatch) -> None:
    f8.install(monkeypatch)
    for name in ("gemm_fp8_blocks", "quant_blocks_fp8", "EPI_BIAS_GELU_TANH_FP8"):
        monkeypatch.setattr(base, name, globals()[name], raising=False)


def quant_blocks(x: torch.Tensor, block: int = 128):
    """fp32 [rows, K] -> (e4m3 codes [rows, K], fp32 scales [rows, K / block])."""
    rows, K = x.shape
    xb = x.float().reshape(rows, K // block, block)
    amax = xb.abs().amax(-1)
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (xb / s[..., None]).clamp(-448.0, 448.0).to(E4M3).reshape(rows, K), s


def quant_blocks_fp8(x, *, block: int = 128, out=None, out_scale=None):
    base._need(x, torch.bfloat16, "x")
    if x.dim() != 2:
        raise OsbError(f"quant_blocks_fp8: x must be [rows, K], got {tuple(x.shape)}")
    rows, K = x.shape
    if K % 128 or block not in (128, K):
        raise OsbError(f"osb_quant_blocks_fp8 failed (-1): K must be a positive multiple of 128 and block 128 or K "
                       f"(K {K} block {block})")
    if x.stride(0) % 8:
        raise OsbError("osb_quant_blocks_fp8 failed (-1): ldx must be a multiple of 8")
    q, s = quant_blocks(x, block)
    base._count("quant_blocks_fp8", (rows, K, block))
    return f8._put(q, out), f8._put(s, out_scale)


def gemm_fp8_blocks(a8, a_scale, w8, w_scale, bias=None, *, epilogue: int = base.EPI_BIAS, residual=None, gate=None,
                    group_rows: int = 0, mod_index=None, out=None, out_scale=None, block_n: int = 0):
    base._need(a8, E4M3, "a8"); base._need(w8, E4M3, "w8")
    base._need(a_scale, torch.float32, "a_scale"); base._need(w_scale, torch.float32, "w_scale")
    for t, n in ((bias, "bias"), (residual, "residual")):
        base._need(t, torch.bfloat16, n)
    base._need(gate, torch.float32, "gate"); base._need(mod_index, torch.int32, "mod_index")
    if a8.dim() != 2 or w8.dim() != 2 or a8.shape[1] != w8.shape[1]:
        raise OsbError(f"gemm_fp8_blocks: a8 [M, K] and w8 [N, K] expected, got {tuple(a8.shape)} and {tuple(w8.shape)}")
    M, K = a8.shape
    N = w8.shape[0]
    if K % 128:
        raise OsbError(f"osb_gemm_fp8_blocks failed (-1): K must be a multiple of 128 (one e4m3 k-block), got {K}")
    if N % 8:
        raise OsbError(f"osb_gemm_fp8_blocks failed (-1): N must be a multiple of 8, got {N}")
    KB = K // 128
    if a_scale is None or w_scale is None or w_scale.shape != (N,) or a_scale.shape not in ((M,), (M, KB)):
        raise OsbError(f"gemm_fp8_blocks: a_scale must be [{M}] or [{M}, {KB}] and w_scale [{N}]")
    base._epilogue_shapes("gemm_fp8_blocks", M, N, N, out, bias, residual, gate, group_rows, mod_index)
    fp8_out = epilogue == EPI_BIAS_GELU_TANH_FP8
    if fp8_out and out_scale is not None and tuple(out_scale.shape) != (M, N // 128):
        raise OsbError(f"out_scale must be a float32 [{M}, {N // 128}] tensor (row stride free)")
    if block_n not in ((0, 128) if fp8_out else (0, 64, 128)):
        raise OsbError(f"osb_gemm_fp8_blocks failed (-3): unsupported block_n {block_n}")
    if not (fp8_out or base.EPI_BIAS <= epilogue <= base.EPI_BIAS_GATE_RES):
        raise OsbError(f"osb_gemm_fp8_blocks failed (-1): epilogue {epilogue} is not built for FP8")
    if fp8_out and N % 128:
        raise OsbError(f"osb_gemm_fp8_blocks failed (-1): the FP8 GELU epilogue needs N % 128 == 0, got {N}")
    dt = base.ACC_DTYPE
    sa = a_scale.to(dt)[:, None].expand(M, KB) if a_scale.dim() == 1 else a_scale.to(dt)
    a, w = a8.to(dt), w8.to(dt)
    acc = torch.zeros(M, N, dtype=dt, device=a8.device)
    for kb in range(KB):
        k = slice(128 * kb, 128 * kb + 128)
        acc = acc + (a[:, k] @ w[:, k].t()) * sa[:, kb:kb + 1]
    acc = acc * w_scale.to(dt)
    if bias is not None:
        acc = acc + bias.to(dt)
    base._count("gemm_fp8_blocks", (M, N, K, epilogue, a_scale.dim()))
    if fp8_out:
        q, s = quant_blocks(F.gelu(acc, approximate="tanh").float())
        return f8._put(q, out), f8._put(s, out_scale)
    if epilogue == base.EPI_BIAS_GELU_TANH:
        acc = F.gelu(acc, approximate="tanh")
    elif epilogue == base.EPI_BIAS_GATE_RES:
        if gate is not None:
            acc = acc * gate[base._groups(M, group_rows if group_rows > 0 else M, mod_index, a8.device)].to(dt)
        if residual is not None:
            acc = acc + residual.to(dt)
    base._need(out, torch.bfloat16, "out")
    return f8._put(acc.to(torch.bfloat16), out)

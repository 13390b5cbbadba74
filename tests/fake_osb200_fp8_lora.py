"""FP8 LoRA entry of the CPU stand-in of the `osb200` binding (TEST INFRASTRUCTURE, not a fallback): a torch restatement
of `gemm_fp8_lora` (include/osb200.h, osb_gemm_fp8_lora) with the kernel's refusals and the launch-count convention of
tests/fake_osb200.py, layered on tests/fake_osb200_fp8_blocks.py.

The arithmetic follows the kernel's, in `fake_osb200.ACC_DTYPE`: each 128-element k-block's e4m3 partial times
a_scale[m, kb] is added into the accumulator; the accumulator is multiplied by w_scale[n] (the FP8 sum only); each
64-column k-block of the rank tail adds its partial U[:, j] B[:, j]^T unscaled; col_scale (DoRA, None = 1) multiplies the
total; then the bias, the epilogue and one rounding (bf16, or the block rule of the FP8 GELU epilogue).

`install(monkeypatch)` adds this entry (and those of the block-scaled FP8 stand-in) to tests/fake_osb200.py for one
test; `install_fp8_proj` does the same on top of the FP8 projection stand-ins (tests/fake_osb200_fp8_proj.py)."""
import torch
import torch.nn.functional as F

from tests import fake_osb200 as base
from tests import fake_osb200_fp8 as f8
from tests import fake_osb200_fp8_blocks as FB

OsbError = base.OsbError
E4M3 = torch.float8_e4m3fn


def install(monkeypatch) -> None:
    FB.install(monkeypatch)
    monkeypatch.setattr(base, "gemm_fp8_lora", gemm_fp8_lora, raising=False)


def install_fp8_proj(monkeypatch) -> None:
    from tests import fake_osb200_fp8_proj as FP

    FP.install(monkeypatch)
    monkeypatch.setattr(base, "gemm_fp8_lora", gemm_fp8_lora, raising=False)


def gemm_fp8_lora_acc(a8, a_scale, w8, w_scale, u, b, col_scale=None, dt=torch.float32):
    """g * (w_scale * sum_kb a_scale[:, kb] * acc_kb + sum over 64-column tail blocks of u b^T), accumulated in `dt`."""
    M, K = a8.shape
    KB = K // 128
    sa = a_scale.to(dt)[:, None].expand(M, KB) if a_scale.dim() == 1 else a_scale.to(dt)
    a, w = a8.to(dt), w8.to(dt)
    acc = torch.zeros(M, w8.shape[0], dtype=dt, device=a8.device)
    for kb in range(KB):
        k = slice(128 * kb, 128 * kb + 128)
        acc = acc + (a[:, k] @ w[:, k].t()) * sa[:, kb:kb + 1]
    acc = acc * w_scale.to(dt)
    uu, bb = u.to(dt), b.to(dt)
    for j0 in range(0, u.shape[1], 64):
        acc = acc + uu[:, j0:j0 + 64] @ bb[:, j0:j0 + 64].t()
    if col_scale is not None:
        acc = acc * col_scale.to(dt)
    return acc


def gemm_fp8_lora(a8, a_scale, w8, w_scale, bias, u, b, *, epilogue: int = base.EPI_BIAS, residual=None, gate=None,
                  group_rows: int = 0, mod_index=None, out=None, out_scale=None, block_n: int = 0, col_scale=None):
    base._need(a8, E4M3, "a8"); base._need(w8, E4M3, "w8")
    base._need(a_scale, torch.float32, "a_scale"); base._need(w_scale, torch.float32, "w_scale")
    for t, n in ((bias, "bias"), (residual, "residual"), (u, "u"), (b, "b")):
        base._need(t, torch.bfloat16, n)
    base._need(gate, torch.float32, "gate"); base._need(mod_index, torch.int32, "mod_index")
    if a8.dim() != 2 or w8.dim() != 2 or a8.shape[1] != w8.shape[1]:
        raise OsbError(f"gemm_fp8_lora: a8 [M, K] and w8 [N, K] expected, got {tuple(a8.shape)} and {tuple(w8.shape)}")
    M, K = a8.shape
    N = w8.shape[0]
    if u is None or b is None or u.dim() != 2 or b.dim() != 2 or u.shape[0] != M or b.shape[0] != N \
            or u.shape[1] != b.shape[1]:
        raise OsbError(f"gemm_fp8_lora: u must be [M, r] and b [N, r] for a {M} x {N} GEMM")
    r = u.shape[1]
    if col_scale is not None and (col_scale.dtype != torch.float32 or col_scale.shape != (N,)
                                  or not col_scale.is_contiguous() or col_scale.device != a8.device):
        raise OsbError(f"gemm_fp8_lora: col_scale must be a contiguous float32 [{N}] tensor on {a8.device}")
    if K % 128:
        raise OsbError(f"osb_gemm_fp8_lora failed (-1): K must be a multiple of 128 (one e4m3 k-block), got {K}")
    if N % 8:
        raise OsbError(f"osb_gemm_fp8_lora failed (-1): N must be a multiple of 8, got {N}")
    if r <= 0 or r % 8:
        raise OsbError(f"osb_gemm_fp8_lora failed (-1): rank r must be a positive multiple of 8, got {r}")
    if u.stride(0) % 8 or b.stride(0) % 8:
        raise OsbError("osb_gemm_fp8_lora failed (-1): ldu and ldb must be multiples of 8")
    KB = K // 128
    if w_scale.shape != (N,) or a_scale.shape not in ((M,), (M, KB)):
        raise OsbError(f"gemm_fp8_lora: a_scale must be [{M}] or [{M}, {KB}] and w_scale [{N}]")
    base._epilogue_shapes("gemm_fp8_lora", M, N, N, out, bias, residual, gate, group_rows, mod_index)
    fp8_out = epilogue == FB.EPI_BIAS_GELU_TANH_FP8
    if fp8_out and out_scale is not None and tuple(out_scale.shape) != (M, N // 128):
        raise OsbError(f"out_scale must be a float32 [{M}, {N // 128}] tensor (row stride free)")
    if block_n not in ((0, 128) if fp8_out else (0, 64, 128)):
        raise OsbError(f"osb_gemm_fp8_lora failed (-3): unsupported block_n {block_n}")
    if not (fp8_out or base.EPI_BIAS <= epilogue <= base.EPI_BIAS_GATE_RES):
        raise OsbError(f"osb_gemm_fp8_lora failed (-1): epilogue {epilogue} is not built for FP8")
    if fp8_out and N % 128:
        raise OsbError(f"osb_gemm_fp8_lora failed (-1): the FP8 GELU epilogue needs N % 128 == 0, got {N}")
    dt = base.ACC_DTYPE
    acc = gemm_fp8_lora_acc(a8, a_scale, w8, w_scale, u, b, col_scale, dt)
    if bias is not None:
        acc = acc + bias.to(dt)
    base._count("gemm_fp8_lora", (M, N, K, r, epilogue, a_scale.dim()))
    if fp8_out:
        q, s = FB.quant_blocks(F.gelu(acc, approximate="tanh").float())
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

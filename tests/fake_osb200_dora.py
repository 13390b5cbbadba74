"""DoRA entry of the CPU stand-in of the `osb200` binding (TEST INFRASTRUCTURE, not a fallback): `gemm_lora` with the
`col_scale` argument of include/osb200.h osb_gemm_lora, restated in torch.  The accumulator a w^T + u b^T is multiplied
by col_scale[n] before the bias and the epilogue, with one rounding to bf16; without col_scale it is the computation of
tests/lora_ref.py::gemm_lora, and both log the same "gemm_lora" launch, so launch lists compare across them.

`install(monkeypatch)` puts this `gemm_lora` on tests/fake_osb200.py for the duration of one test, the way
tests/fake_osb200_fp8.py adds the FP8 entries."""
import torch
import torch.nn.functional as F

from tests import fake_osb200 as base


def install(monkeypatch) -> None:
    monkeypatch.setattr(base, "gemm_lora", gemm_lora, raising=False)


def gemm_dora_fp32(a, w, bias, u, b, *, col_scale=None, epilogue=base.EPI_BIAS, residual=None, gate=None, group_rows=0,
                   mod_index=None, acc_dtype=torch.float32):
    """epilogue(col_scale * (a w^T + u b^T) + bias) before the rounding to bf16, accumulated in `acc_dtype`."""
    M = a.shape[0]
    acc = a.to(acc_dtype) @ w.to(acc_dtype).t() + u.to(acc_dtype) @ b.to(acc_dtype).t()
    if col_scale is not None:
        acc = acc * col_scale.to(acc_dtype)
    if bias is not None:
        acc = acc + bias.to(acc_dtype)
    if epilogue == base.EPI_BIAS_GELU_TANH:
        acc = F.gelu(acc, approximate="tanh")
    elif epilogue == base.EPI_BIAS_GATE_RES:
        if gate is not None:
            acc = acc * gate.to(acc_dtype)[base._groups(M, group_rows if group_rows > 0 else M, mod_index, a.device)]
        if residual is not None:
            acc = acc + residual.to(acc_dtype)
    return acc


def gemm_lora(a, w, bias, u, b, *, epilogue=base.EPI_BIAS, residual=None, gate=None, group_rows=0, mod_index=None,
              out=None, block_n=0, col_scale=None):
    for t, n in ((a, "a"), (w, "w"), (bias, "bias"), (u, "u"), (b, "b"), (residual, "residual"), (out, "out")):
        base._need(t, torch.bfloat16, n)
    base._need(gate, torch.float32, "gate"); base._need(mod_index, torch.int32, "mod_index")
    if a.dim() != 2 or w.dim() != 2 or a.shape[1] != w.shape[1]:
        raise base.OsbError(f"gemm_lora: a [M, K] and w [N, K] expected, got {tuple(a.shape)} and {tuple(w.shape)}")
    M, K = a.shape
    N = w.shape[0]
    base._epilogue_shapes("gemm_lora", M, N, N, out, bias, residual, gate, group_rows, mod_index)
    if K % 8 or N % 8:
        raise base.OsbError(f"osb_gemm_lora failed (-1): K and N must be multiples of 8 (K {K} N {N})")
    if u.shape[0] != M or b.shape[0] != N or u.shape[1] != b.shape[1] or u.shape[1] % 8:
        raise base.OsbError(f"gemm_lora: u {tuple(u.shape)} / b {tuple(b.shape)} do not fit a {M} x {N} GEMM with r % 8 == 0")
    if col_scale is not None and (col_scale.dtype != torch.float32 or col_scale.shape != (N,)
                                  or not col_scale.is_contiguous() or col_scale.device != a.device):
        raise base.OsbError(f"gemm_lora: col_scale must be a contiguous float32 [{N}] tensor on {a.device}")
    y = gemm_dora_fp32(a, w, bias, u, b, col_scale=col_scale, epilogue=epilogue, residual=residual, gate=gate,
                       group_rows=group_rows, mod_index=mod_index, acc_dtype=base.ACC_DTYPE).to(torch.bfloat16)
    base._count("gemm_lora", (M, N, K, u.shape[1], epilogue))
    if out is None:
        return y
    out.copy_(y)
    return out

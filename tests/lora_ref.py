"""fp32 restatement of `osb200.gemm_lora` (include/osb200.h osb_gemm_lora): the CPU tests add it to the binding stand-in
(tests/fake_osb200.py) by fixture, and the GPU tests compare the kernel with it on the same bf16 operands."""
import torch
import torch.nn.functional as F

EPI_BIAS, EPI_BIAS_GELU_TANH, EPI_BIAS_GATE_RES = 0, 1, 2


def gemm_lora_fp32(a, w, bias, u, b, *, epilogue=EPI_BIAS, residual=None, gate=None, group_rows=0, mod_index=None,
                   acc_dtype=torch.float32):
    """epilogue(a w^T + u b^T + bias) before the rounding to bf16, accumulated in `acc_dtype`."""
    M = a.shape[0]
    acc = a.to(acc_dtype) @ w.to(acc_dtype).t() + u.to(acc_dtype) @ b.to(acc_dtype).t()
    if bias is not None:
        acc = acc + bias.to(acc_dtype)
    if epilogue == EPI_BIAS_GELU_TANH:
        acc = F.gelu(acc, approximate="tanh")
    elif epilogue == EPI_BIAS_GATE_RES:
        if gate is not None:
            g = torch.arange(M, device=a.device) // (group_rows if group_rows > 0 else M)
            if mod_index is not None:
                g = mod_index.long()[g]
            acc = acc * gate.to(acc_dtype)[g]
        if residual is not None:
            acc = acc + residual.to(acc_dtype)
    return acc


def gemm_lora(a, w, bias, u, b, *, epilogue=EPI_BIAS, residual=None, gate=None, group_rows=0, mod_index=None, out=None,
              block_n=0):
    """The binding's contract on the CPU: same argument checks as `gemm`, one rounding to bf16, `out` may alias
    `residual`.  Logged as a "gemm_lora" launch in the stand-in's call log."""
    from tests import fake_osb200 as F_

    for t, n in ((a, "a"), (w, "w"), (bias, "bias"), (u, "u"), (b, "b"), (residual, "residual"), (out, "out")):
        F_._need(t, torch.bfloat16, n)
    F_._need(gate, torch.float32, "gate"); F_._need(mod_index, torch.int32, "mod_index")
    if a.dim() != 2 or w.dim() != 2 or a.shape[1] != w.shape[1]:
        raise F_.OsbError(f"gemm_lora: a [M, K] and w [N, K] expected, got {tuple(a.shape)} and {tuple(w.shape)}")
    M, K = a.shape
    N = w.shape[0]
    F_._epilogue_shapes("gemm_lora", M, N, N, out, bias, residual, gate, group_rows, mod_index)
    if K % 8 or N % 8:
        raise F_.OsbError(f"osb_gemm_lora failed (-1): K and N must be multiples of 8 (K {K} N {N})")
    if u.shape[0] != M or b.shape[0] != N or u.shape[1] != b.shape[1] or u.shape[1] % 8:
        raise F_.OsbError(f"gemm_lora: u {tuple(u.shape)} / b {tuple(b.shape)} do not fit a {M} x {N} GEMM with r % 8 == 0")
    y = gemm_lora_fp32(a, w, bias, u, b, epilogue=epilogue, residual=residual, gate=gate, group_rows=group_rows,
                       mod_index=mod_index, acc_dtype=F_.ACC_DTYPE).to(torch.bfloat16)
    F_._count("gemm_lora", (M, N, K, u.shape[1], epilogue))
    if out is None:
        return y
    out.copy_(y)
    return out

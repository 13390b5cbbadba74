"""Text-encoder entries of the CPU stand-in of the `osb200` binding (TEST INFRASTRUCTURE, not a fallback): torch
restatements of `attn_short_bias`, `rms_norm` and the `EPI_GATED_GELU` / `EPI_BIAS_QUICK_GELU` GEMM epilogues, with the
refusals of the kernels and the launch-count convention of tests/fake_osb200.py (one count per launch, nothing counted
for a refused call).  Rounding points mirror the kernels: fp32 math, one rounding to bf16 per op; RMSNorm rounds twice
as T5LayerNorm does; attention rounds the unnormalised P to bf16 before P V.

`install(monkeypatch)` adds these entries to tests/fake_osb200.py for the duration of one test, so that the host-side
text encoder runs against the stand-in installed by the `fake_osb` fixture; `gemm` keeps the base stand-in's behaviour
for epilogues 0-2.  The module also exposes every name the GPU conformance tests call on it."""
import torch
import torch.nn.functional as F

from tests import fake_osb200 as base

EPI_GATED_GELU, EPI_BIAS_QUICK_GELU = 3, 4
OsbError = base.OsbError
launch_count = base.launch_count
_base_gemm = base.gemm


def install(monkeypatch) -> None:
    for name in ("EPI_GATED_GELU", "EPI_BIAS_QUICK_GELU", "gemm", "rms_norm", "attn_short_bias", "interleave_gated"):
        monkeypatch.setattr(base, name, globals()[name], raising=False)


def interleave_gated(wi_0, wi_1):
    return torch.stack((wi_0, wi_1), dim=1).reshape(2 * wi_0.shape[0], wi_0.shape[1]).contiguous()


def gemm(a, w, bias=None, *, epilogue: int = base.EPI_BIAS, residual=None, gate=None, group_rows: int = 0, mod_index=None,
         out=None, cta_group: int = 0, block_n: int = 0):
    if not base.EPI_BIAS <= epilogue <= EPI_BIAS_QUICK_GELU:
        raise OsbError(f"osb_gemm_bf16 failed (-1): osb_gemm_bf16: unknown epilogue {epilogue}")
    if epilogue <= base.EPI_BIAS_GATE_RES:
        return _base_gemm(a, w, bias, epilogue=epilogue, residual=residual, gate=gate, group_rows=group_rows,
                          mod_index=mod_index, out=out, cta_group=cta_group, block_n=block_n)
    for t, n in ((a, "a"), (w, "w"), (bias, "bias"), (out, "out")):
        base._need(t, torch.bfloat16, n)
    assert a.dim() == 2 and w.dim() == 2 and a.shape[1] == w.shape[1]
    M, K = a.shape
    N = w.shape[0]
    if K % 8 or N % 8:
        raise OsbError(f"osb_gemm_bf16 failed (-1): osb_gemm_bf16: K and N must be multiples of 8 (K {K} N {N})")
    acc = a.to(base.ACC_DTYPE) @ w.to(base.ACC_DTYPE).t()
    if bias is not None:
        acc = acc + bias.to(base.ACC_DTYPE)
    if epilogue == EPI_GATED_GELU:   # rows of w interleave wi_0 (even) and wi_1 (odd)
        acc = F.gelu(acc[:, 0::2], approximate="tanh") * acc[:, 1::2]
    else:
        acc = acc * torch.sigmoid(1.702 * acc)
    if (out.stride(0) if out is not None else acc.shape[1]) % 8:
        raise OsbError("osb_gemm_bf16 failed (-1): osb_gemm_bf16: D must be 16-byte aligned with ldd % 8 == 0")
    y = acc.to(torch.bfloat16)
    base._count("gemm", (M, N, K, epilogue))
    if out is None:
        return y
    out.copy_(y)
    return out


def rms_norm(x, w, *, eps: float = 1e-6, out=None):
    base._need(x, torch.bfloat16, "x"); base._need(w, torch.bfloat16, "w")
    if x.dim() != 2 or not x.is_contiguous() or w.shape != (x.shape[1],):
        raise OsbError(f"rms_norm: x must be a contiguous [rows, C] tensor and w [C], got {tuple(x.shape)} and {tuple(w.shape)}")
    C = x.shape[1]
    if C % 8 or C > 4096:
        raise OsbError(f"osb_rms_norm failed (-1): osb_rms_norm: C must be a multiple of 8 and <= 4096 (got {C})")
    xf = x.float()
    t = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(torch.bfloat16)
    y = (w.float() * t.float()).to(torch.bfloat16)
    base._count("rms_norm", tuple(x.shape))
    if out is None:
        return y
    out.copy_(y)
    return out


def attn_short_bias(q, k, v, out, bias, *, num_seqs: int, seqs_per_batch: int, q_strides, k_strides, Lq: int, Lk: int,
                    num_heads: int, head_dim: int, kv_lens=None, softmax_scale=None):
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        base._need(t, torch.bfloat16, n)
    base._need(bias, torch.float32, "bias"); base._need(kv_lens, torch.int32, "kv_lens")
    H, D = num_heads, head_dim
    n_rel = Lq + Lk - 1
    if bias is None or not bias.is_contiguous() or bias.shape not in ((n_rel,), (H, n_rel)):
        raise OsbError(f"attn_short_bias: bias must be a contiguous fp32 [{n_rel}] or [{H}, {n_rel}] tensor, got "
                       f"{None if bias is None else tuple(bias.shape)}")
    if D != 64:
        raise OsbError(f"osb_attn_short_bias failed (-1): osb_attn_short_bias: head_dim {D} not built (64)")
    dev = q.device
    s = torch.arange(num_seqs, device=dev)
    b, j = s // seqs_per_batch, s % seqs_per_batch

    def rows(strides, L):
        bs, ss, ts = strides
        return (b * bs + j * ss)[:, None] + torch.arange(L, device=dev)[None] * ts

    rq, rk = rows(q_strides, Lq), rows(k_strides, Lk)
    qf = q[rq][..., : H * D].float().view(num_seqs, Lq, H, D).transpose(1, 2)
    kf = k[rk][..., : H * D].float().view(num_seqs, Lk, H, D).transpose(1, 2)
    vf = v[rk][..., : H * D].float().view(num_seqs, Lk, H, D).transpose(1, 2)
    scale = softmax_scale if softmax_scale is not None else D ** -0.5
    rel = torch.arange(Lk, device=dev)[None, :] - torch.arange(Lq, device=dev)[:, None] + Lq - 1
    bb = bias.view(-1, n_rel)[:, rel]                                               # [1 or H, Lq, Lk]
    sc = (qf @ kf.transpose(-1, -2)) * scale + bb[None]
    if kv_lens is not None:
        dead = torch.arange(Lk, device=dev)[None, :] >= kv_lens.long()[:, None]
        sc = sc.masked_fill(dead[:, None, None, :], float("-inf"))
    m = sc.amax(-1, keepdim=True)
    p = torch.exp(sc - torch.where(torch.isinf(m), torch.zeros_like(m), m))
    l = p.sum(-1, keepdim=True)
    o = (p.to(torch.bfloat16).float() @ vf) / torch.where(l > 0, l, torch.ones_like(l))   # P is rounded before P V
    o = o.transpose(1, 2).reshape(num_seqs, Lq, H * D).to(torch.bfloat16)
    out[rq.reshape(-1), : H * D] = o.reshape(-1, H * D)
    base._count("attn_short", (num_seqs, Lq, Lk, H, D, "bias"))
    return out

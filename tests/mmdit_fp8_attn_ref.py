"""FP8-emulation reference of the MMDiT FP8 attention path (include/osb200.h, osb_attn_fp8), for the tests.

The pinned oracle (`oracle/mmdit_oracle.py`), typically run in bf16, with its `attention` replaced by fp32 arithmetic on
dequantized operands, rounded where the product rounds:
- q and k after RMSNorm and RoPE (in the oracle's dtype), per (token, head);
- v per channel over the sequence;
- P as e4m3(256 p) / 256 with p relative to the FINAL row maximum, normalised by the fp32 sum of the unquantized p.
The kernel quantizes P against the running maximum of its 128-key blocks, so this is not its arithmetic bit for bit; it is
the same kind of yardstick the FP8 MLP tests use.  `fp8_attention()` patches the oracle for the duration of a `with`."""
import contextlib

import torch

from tests import fp8_ref as R


def qdq_p(p: torch.Tensor) -> torch.Tensor:
    return R.e4m3_round(256.0 * p).float() / 256.0


def attention_from_operands(q, k, v, scale: float):
    """fp32 softmax attention of dequantized [.., L, D] operands with P quantized as the contract does (final max)."""
    s = (q @ k.transpose(-1, -2)) * scale
    p = torch.exp(s - s.amax(-1, keepdim=True))
    return (qdq_p(p) @ v) / p.sum(-1, keepdim=True)


def _attention(M):
    def attention(q, k, v, pe):
        if isinstance(pe, torch.Tensor):
            q, k = M.apply_rope(q, pe), M.apply_rope(k, pe)
        else:
            q, k = M.apply_rope_rotate_half(q, *pe), M.apply_rope_rotate_half(k, *pe)
        qd, kd = R.qdq(q.float()), R.qdq(k.float())
        vd = R.qdq(v.float().transpose(-1, -2)).transpose(-1, -2)
        o = attention_from_operands(qd, kd, vd, q.shape[-1] ** -0.5)
        return o.to(v.dtype).transpose(1, 2).reshape(q.shape[0], q.shape[2], -1)
    return attention


@contextlib.contextmanager
def fp8_attention():
    """Patch oracle/mmdit_oracle.py so that `model_forward` runs every joint attention at the FP8 rounding points."""
    from oracle import mmdit_oracle as M

    saved = M.attention
    M.attention = _attention(M)
    try:
        yield M
    finally:
        M.attention = saved


def operands_cpu(B, L, H, seed=0, split=None, liger=True):
    g = torch.Generator().manual_seed(seed)
    C = H * 128
    qkv = (torch.randn(B * L, 3 * C, generator=g) * 2).to(torch.bfloat16)
    qkv[3, 2 * C:2 * C + 5] = 40.0                      # a v column with one large entry
    qkv[:, 2 * C + 7] = 0.0                             # an all-zero v column: scale 1, codes 0
    w = [(1 + 0.3 * torch.randn(128, generator=g)).to(torch.bfloat16) for _ in range(4)]
    ang = torch.randn(L, 64, generator=g)
    kw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H,
              head_dim=128, q_norm_w=w[0], k_norm_w=w[1], rope_cos=torch.cos(ang), rope_sin=torch.sin(ang),
              rope_half=liger, q_norm_w2=None, k_norm_w2=None, norm_split=0)
    if split is not None:
        kw.update(q_norm_w2=w[2], k_norm_w2=w[3], norm_split=split)
    return qkv, kw


def operands_cuda(B, L, H, liger, split, seed=0, wscale=0.3, wmean=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = H * 128
    qkv = (torch.randn(B * L, 3 * C, device="cuda", generator=g) * 2).to(torch.bfloat16)
    w = [(wmean + wscale * torch.randn(128, device="cuda", generator=g)).to(torch.bfloat16) for _ in range(4)]
    ang = torch.rand(L, 64, device="cuda", generator=g) * 6.28
    kw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H,
              head_dim=128, q_norm_w=w[0], k_norm_w=w[1], rope_cos=torch.cos(ang), rope_sin=torch.sin(ang),
              rope_half=liger, q_norm_w2=None, k_norm_w2=None, norm_split=0)
    if split is not None:
        kw.update(q_norm_w2=w[2], k_norm_w2=w[3], norm_split=split)
    return qkv, kw

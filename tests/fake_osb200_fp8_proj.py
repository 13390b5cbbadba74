"""Block-scaled e4m3 output of the FP8 attention in the CPU stand-in of the `osb200` binding (TEST INFRASTRUCTURE, not a
fallback): a torch restatement of `attn_fp8_blocks` (include/osb200.h, osb_attn_fp8_blocks) with the kernel's refusals
and the launch-count convention of tests/fake_osb200.py.

The attention is that of tests/fake_osb200_fp8_attn.py up to the fp32 value v = O s_v / (256 l); each (row, head) of v
is then one 1 x 128 block of the block rule of tests/fake_osb200_fp8_blocks.py (s = amax / 448, 1 for a zero block,
codes = the float8_e4m3fn cast of v / s).  Codes and scales go to column slices with a free row stride.

`install(monkeypatch)` adds this entry, and those of the FP8 attention and block-scaled FP8 stand-ins, to
tests/fake_osb200.py for one test."""
import torch

from tests import fake_osb200 as base
from tests import fake_osb200_fp8_attn as FA
from tests import fake_osb200_fp8_blocks as FB

OsbError = base.OsbError
E4M3 = torch.float8_e4m3fn


def install(monkeypatch) -> None:
    FA.install(monkeypatch)
    FB.install(monkeypatch)
    monkeypatch.setattr(base, "attn_fp8_blocks", attn_fp8_blocks, raising=False)


def attn_fp8_blocks(q, k, v, out, out_scale, *, workspace, num_seqs: int, seqs_per_batch: int, q_strides, k_strides,
                    Lq: int, Lk: int, num_heads: int, head_dim: int, kv_lens=None, q_norm_w=None, k_norm_w=None,
                    norm_eps: float = 1e-6, rope_cos=None, rope_sin=None, softmax_scale=None, q_norm_w2=None,
                    k_norm_w2=None, norm_split: int = 0, impl: int = 0, rope_half: bool = False):
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (q_norm_w, "q_norm_w"), (k_norm_w, "k_norm_w")):
        base._need(t, torch.bfloat16, n)
    base._need(out, E4M3, "out"); base._need(out_scale, torch.float32, "out_scale")
    base._need(rope_cos, torch.float32, "rope_cos"); base._need(rope_sin, torch.float32, "rope_sin")
    for t, n, w in ((out, "out", num_heads * head_dim), (out_scale, "out_scale", num_heads)):
        if t is None or t.dim() != 2 or t.stride(1) != 1 or t.shape[1] < w:
            raise OsbError(f"attn_fp8_blocks: {n} must be a 2-D tensor of >= {w} unit-stride columns")
    if head_dim != 128:
        raise OsbError(f"osb_attn_fp8_blocks failed (-1): osb_attn_fp8_blocks: head_dim {head_dim} not built (128)")
    if Lq != Lk:
        raise OsbError(f"osb_attn_fp8_blocks failed (-1): osb_attn_fp8_blocks: self-attention only (Lq {Lq} != Lk {Lk})")
    if kv_lens is not None:
        raise OsbError("osb_attn_fp8_blocks failed (-1): osb_attn_fp8_blocks: kv_lens is not supported")
    if seqs_per_batch != 1:
        raise OsbError("osb_attn_fp8_blocks failed (-1): osb_attn_fp8_blocks: one sequence per batch element")
    if out.stride(0) % 8:
        raise OsbError("osb_attn_fp8_blocks failed (-1): leading dimensions must be multiples of 8 elements")
    if not isinstance(workspace, FA.AttnFp8Workspace):
        raise OsbError("attn_fp8_blocks: workspace must come from attn_fp8_workspace()")
    L, H = Lq, num_heads
    Lp = -(-L // FA.ATTN_FP8_KEY_BLOCK) * FA.ATTN_FP8_KEY_BLOCK
    if num_seqs * H > workspace.s_v.shape[0] or Lp > workspace.Lpad:
        raise OsbError("osb_attn_fp8_blocks failed (-1): workspace too small")
    qf, kf, vf, rq = FA.stage(q, k, v, num_seqs=num_seqs, q_strides=q_strides, k_strides=k_strides, L=L, H=H,
                              q_norm_w=q_norm_w, k_norm_w=k_norm_w, norm_eps=norm_eps, rope_cos=rope_cos,
                              rope_sin=rope_sin, q_norm_w2=q_norm_w2, k_norm_w2=k_norm_w2, norm_split=norm_split,
                              rope_half=rope_half)
    FA.fill_workspace(workspace, qf, kf, vf)
    scale = softmax_scale if softmax_scale is not None else head_dim ** -0.5
    o = FA.attention_from_workspace(workspace, num_seqs * H, L, scale)
    o = o.view(num_seqs, H, L, 128).transpose(1, 2).reshape(num_seqs * L, H * 128)
    codes, s = FB.quant_blocks(o)
    rows = rq.reshape(-1)
    out[rows, : H * 128] = codes
    out_scale[rows, :H] = s
    base._count("attn_fp8_blocks", (num_seqs, L, H), launches=3)
    return out, out_scale

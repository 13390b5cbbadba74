"""FP8 attention entries of the CPU stand-in of the `osb200` binding (TEST INFRASTRUCTURE, not a fallback): a torch
restatement of `attn_fp8` and its workspace (include/osb200.h, osb_attn_fp8) with the kernel's refusals and the
launch-count convention of tests/fake_osb200.py.

- q~ / k~: the bf16 rows osb_attn_short stages (fp32 RMSNorm with the stream's weight, RoPE, one rounding); per (token,
  head) s = amax / 448 (1 for a zero row), codes = the torch float8_e4m3fn cast of x / s (round to nearest even).
- v: per channel over the sequence, the same rule along the tokens.
- The workspace is filled in the header's layout: q8 / k8 [B*H, Lpad, 128] with zero codes and scale 1 past L, vt8
  [B*H, 128, Lpad] with key j(p) at position p of every 32-key group (`vt8_key`).
- Attention is computed from the workspace operands as the kernel does: key blocks of 128, scores in log2 units, online
  maximum, P8 = e4m3(256 p), partial P8 V8 promoted as O = alpha O + partial, out = O s_v / (256 l).

`install(monkeypatch)` adds these entries to tests/fake_osb200.py for one test."""
import math

import torch

from tests import fake_osb200 as base

OsbError = base.OsbError
E4M3 = torch.float8_e4m3fn
ATTN_FP8_KEY_BLOCK = 128


def install(monkeypatch) -> None:
    for name in ("attn_fp8", "attn_fp8_workspace", "AttnFp8Workspace", "ATTN_FP8_KEY_BLOCK"):
        monkeypatch.setattr(base, name, globals()[name], raising=False)


def vt8_key(pos: torch.Tensor) -> torch.Tensor:
    """Key held at position `pos` of vt8 (include/osb200.h): j(p) = 16 (p/16) + 2 ((p%16)/4) + p%2 + 8 ((p%4)/2) inside
    each 32-key group."""
    return (pos & ~31) + 16 * ((pos >> 4) & 1) + 2 * ((pos >> 2) & 3) + (pos & 1) + 8 * ((pos >> 1) & 1)


def _e4m3(x):
    return x.clamp(-448.0, 448.0).to(E4M3)


def _scale(amax):
    # divide by a tensor: on CUDA, torch divides by a Python scalar through its rounded reciprocal
    return torch.where(amax > 0, amax / torch.tensor(448.0, device=amax.device), torch.ones_like(amax))


class AttnFp8Workspace:
    def __init__(self, B: int, L: int, H: int, device):
        BH, Lp = B * H, -(-L // ATTN_FP8_KEY_BLOCK) * ATTN_FP8_KEY_BLOCK
        self.B, self.L, self.H, self.Lpad = B, L, H, Lp
        self.q8 = torch.empty(BH, Lp, 128, dtype=E4M3, device=device)
        self.k8 = torch.empty(BH, Lp, 128, dtype=E4M3, device=device)
        self.vt8 = torch.empty(BH, 128, Lp, dtype=E4M3, device=device)
        self.s_q = torch.empty(BH, Lp, device=device)
        self.s_k = torch.empty(BH, Lp, device=device)
        self.s_v = torch.empty(BH, 128, device=device)
        self.v_amax = torch.zeros(BH, 128, device=device)


def attn_fp8_workspace(B: int, L: int, H: int, device) -> AttnFp8Workspace:
    return AttnFp8Workspace(B, L, H, device)


def stage(q, k, v, *, num_seqs, q_strides, k_strides, L, H, q_norm_w, k_norm_w, norm_eps, rope_cos, rope_sin, q_norm_w2,
          k_norm_w2, norm_split, rope_half):
    """(q~, k~, v) as fp32 [num_seqs, H, L, 128] and the [num_seqs, L] output rows, as osb_attn_short stages them."""
    D, dev = 128, q.device
    b = torch.arange(num_seqs, device=dev)

    def rows(strides):
        bs, _, ts = strides
        return (b * bs)[:, None] + torch.arange(L, device=dev)[None] * ts

    rq, rk = rows(q_strides), rows(k_strides)
    qf = q[rq][..., : H * D].float().view(num_seqs, L, H, D).transpose(1, 2)
    kf = k[rk][..., : H * D].float().view(num_seqs, L, H, D).transpose(1, 2)
    vf = v[rk][..., : H * D].float().view(num_seqs, L, H, D).transpose(1, 2)
    if q_norm_w is not None:
        def normed(x, w, w2):
            y = base._rms(x, w.float(), norm_eps)
            if w2 is not None:
                sel = (torch.arange(L, device=dev) >= norm_split)[None, None, :, None]
                y = torch.where(sel, base._rms(x, w2.float(), norm_eps), y)
            return y
        qf, kf = normed(qf, q_norm_w, q_norm_w2), normed(kf, k_norm_w, k_norm_w2)
    if rope_cos is not None:
        rot = base._rope_half if rope_half else base._rope_interleaved
        qf, kf = rot(qf, rope_cos[:L], rope_sin[:L]), rot(kf, rope_cos[:L], rope_sin[:L])
    return qf.to(torch.bfloat16).float(), kf.to(torch.bfloat16).float(), vf, rq


def fill_workspace(ws: AttnFp8Workspace, qf, kf, vf) -> None:
    """Quantize staged [n, H, L, 128] operands into `ws` in the header's layout."""
    n, H, L, D = qf.shape
    BH, Lp = n * H, -(-L // ATTN_FP8_KEY_BLOCK) * ATTN_FP8_KEY_BLOCK
    views = dict(q8=(BH, Lp, D), k8=(BH, Lp, D), vt8=(BH, D, Lp), s_q=(BH, Lp), s_k=(BH, Lp), s_v=(BH, D))
    t = {name: getattr(ws, name).view(-1)[:math.prod(shape)].view(shape) for name, shape in views.items()}
    for name, x in (("q", qf), ("k", kf)):
        s = _scale(x.abs().amax(-1)).reshape(BH, L)
        codes = _e4m3(x.reshape(BH, L, D) / s[..., None])
        t[name + "8"].zero_()
        t[name + "8"][:, :L] = codes
        t["s_" + name].fill_(1.0)
        t["s_" + name][:, :L] = s
    sv = _scale(vf.abs().amax(2)).reshape(BH, D)
    v8 = torch.zeros(BH, Lp, D, dtype=E4M3, device=vf.device)
    v8[:, :L] = _e4m3(vf.reshape(BH, L, D) / sv[:, None, :])
    t["s_v"].copy_(sv)
    t["vt8"].copy_(v8[:, vt8_key(torch.arange(Lp, device=vf.device))].transpose(1, 2))


def workspace_operands(ws: AttnFp8Workspace, BH: int, L: int):
    """(q8, s_q, k8, s_k, v8 in key order, s_v) of the first BH sequence-heads, read back from the workspace."""
    Lp = -(-L // ATTN_FP8_KEY_BLOCK) * ATTN_FP8_KEY_BLOCK
    q8 = ws.q8.view(-1)[:BH * Lp * 128].view(BH, Lp, 128)
    k8 = ws.k8.view(-1)[:BH * Lp * 128].view(BH, Lp, 128)
    vt8 = ws.vt8.view(-1)[:BH * 128 * Lp].view(BH, 128, Lp)
    v8 = torch.empty(BH, Lp, 128, dtype=E4M3, device=vt8.device)
    v8[:, vt8_key(torch.arange(Lp, device=vt8.device))] = vt8.transpose(1, 2)
    return (q8, ws.s_q.view(-1)[:BH * Lp].view(BH, Lp), k8, ws.s_k.view(-1)[:BH * Lp].view(BH, Lp), v8,
            ws.s_v.view(-1)[:BH * 128].view(BH, 128))


def attention_from_workspace(ws: AttnFp8Workspace, BH: int, L: int, softmax_scale: float) -> torch.Tensor:
    """fp32 [BH, L, 128] output of the contract's online FP8 attention, from the workspace operands."""
    q8, sq, k8, sk, v8, sv = workspace_operands(ws, BH, L)
    sc = softmax_scale * 1.4426950408889634
    qd, kd, vd = q8[:, :L].float(), k8.float(), v8.float()
    m = torch.full((BH, L, 1), float("-inf"), device=q8.device)
    l = torch.zeros(BH, L, 1, device=q8.device)
    o = torch.zeros(BH, L, 128, device=q8.device)
    for k0 in range(0, L, ATTN_FP8_KEY_BLOCK):
        blk = slice(k0, k0 + ATTN_FP8_KEY_BLOCK)
        s = (qd @ kd[:, blk].transpose(1, 2)) * (sq[:, :L, None] * sc) * sk[:, None, blk]
        s = s.masked_fill(torch.arange(k0, k0 + ATTN_FP8_KEY_BLOCK, device=q8.device) >= L, float("-inf"))
        mn = torch.maximum(m, s.amax(-1, keepdim=True))
        alpha = torch.exp2(m - mn)
        p = torch.exp2(s - mn)
        l = l * alpha + p.sum(-1, keepdim=True)
        o = o * alpha + _e4m3(256.0 * p).float() @ vd[:, blk]
        m = mn
    return o * sv[:, None, :] / (256.0 * l)


def attn_fp8(q, k, v, out, *, workspace, num_seqs: int, seqs_per_batch: int, q_strides, k_strides, Lq: int, Lk: int,
             num_heads: int, head_dim: int, kv_lens=None, q_norm_w=None, k_norm_w=None, norm_eps: float = 1e-6,
             rope_cos=None, rope_sin=None, softmax_scale=None, q_norm_w2=None, k_norm_w2=None, norm_split: int = 0,
             impl: int = 0, rope_half: bool = False):
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out"), (q_norm_w, "q_norm_w"), (k_norm_w, "k_norm_w")):
        base._need(t, torch.bfloat16, n)
    base._need(rope_cos, torch.float32, "rope_cos"); base._need(rope_sin, torch.float32, "rope_sin")
    if head_dim != 128:
        raise OsbError(f"osb_attn_fp8 failed (-1): osb_attn_fp8: head_dim {head_dim} not built (128)")
    if Lq != Lk:
        raise OsbError(f"osb_attn_fp8 failed (-1): osb_attn_fp8: self-attention only (Lq {Lq} != Lk {Lk})")
    if kv_lens is not None:
        raise OsbError("osb_attn_fp8 failed (-1): osb_attn_fp8: kv_lens is not supported")
    if seqs_per_batch != 1:
        raise OsbError("osb_attn_fp8 failed (-1): osb_attn_fp8: one sequence per batch element")
    if (q_norm_w is None) != (k_norm_w is None) or (rope_cos is None) != (rope_sin is None):
        raise OsbError("osb_attn_fp8 failed (-1): norm weights / rope tables must come in pairs")
    if (q_norm_w2 is None) != (k_norm_w2 is None) or (q_norm_w2 is not None and q_norm_w is None):
        raise OsbError("osb_attn_fp8 failed (-1): the second norm weight pair needs the first")
    if not isinstance(workspace, AttnFp8Workspace):
        raise OsbError("attn_fp8: workspace must come from attn_fp8_workspace()")
    L, H = Lq, num_heads
    Lp = -(-L // ATTN_FP8_KEY_BLOCK) * ATTN_FP8_KEY_BLOCK
    if num_seqs * H > workspace.s_v.shape[0] or Lp > workspace.Lpad:
        raise OsbError("osb_attn_fp8 failed (-1): workspace too small")
    qf, kf, vf, rq = stage(q, k, v, num_seqs=num_seqs, q_strides=q_strides, k_strides=k_strides, L=L, H=H,
                           q_norm_w=q_norm_w, k_norm_w=k_norm_w, norm_eps=norm_eps, rope_cos=rope_cos, rope_sin=rope_sin,
                           q_norm_w2=q_norm_w2, k_norm_w2=k_norm_w2, norm_split=norm_split, rope_half=rope_half)
    fill_workspace(workspace, qf, kf, vf)
    scale = softmax_scale if softmax_scale is not None else head_dim ** -0.5
    o = attention_from_workspace(workspace, num_seqs * H, L, scale)
    o = o.view(num_seqs, H, L, 128).transpose(1, 2).reshape(num_seqs * L, H * 128).to(torch.bfloat16)
    out[rq.reshape(-1), : H * 128] = o
    base._count("attn_fp8", (num_seqs, L, H), launches=3)
    return out

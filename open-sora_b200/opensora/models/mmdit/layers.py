"""MMDiT layers on the osb200 kernels — same classes, constructor arguments, state-dict keys and the same
block-`processor` plug-in hook as the reference's `opensora/models/mmdit/layers.py`
(`DoubleStreamBlock.set_processor / forward = self.processor(self, img, txt, vec, pe)` :295-306,
`SingleStreamBlock` :378-388).  The nn.Modules hold parameters; the two processor classes below ARE the drop-in:
they read the block's own parameters and run every FLOP on libosb200 (sm_90a):

  LN(no affine)+modulate -> `osb_ln_modulate`; every Linear -> `osb_gemm_bf16` (bias / GELU-tanh / gate*x+residual
  epilogues); QK-RMSNorm + RoPE + joint txt|img softmax attention -> `osb_attn_short` (per-stream norm weights via
  `norm_split`); `linear2(cat(attn, gelu(mlp)))` reads ONE [rows, 5C] buffer that the attention kernel and the
  GELU GEMM wrote side by side (no torch.cat materialisation, SURVEY.md §2.2 K9).

Any joint sequence length (the flash attention variant streams key blocks), both RoPE layouts (`EmbedND`
interleaved pairs and `LigerEmbedND` rotate-half) and both QKV checkpoint layouts (`fused_qkv` True / False).

LoRA (opensora/utils/lora.py): every Linear is read through `linear_parts` / `lora_pack`, which also return the active
adapter's (A, scaling * B, DoRA column scale or None), if any.  Linears that read one input share one down GEMM
U = x A_cat^T; each output weight then runs `osb_gemm_lora` (g * (x W^T + U B^T) in one accumulator, g = 1 without
DoRA).  Without an adapter the launches are those of the plain model.

FP8 (MMDiTModel.enable_fp8): the MLPs run on e4m3 operands.  Double blocks: ln_modulate_fp8 -> fc1 on
`osb_gemm_fp8_blocks` whose GELU epilogue emits e4m3 codes with 1 x 128 block scales -> fc2 on block-scaled A (gate +
residual).  Single blocks: the qkv part of linear1 stays bf16; the mlp part runs on ln_modulate_fp8 and its GELU epilogue
writes columns C.. of an e4m3 [rows, 5C] cat buffer, `osb_quant_blocks_fp8` fills columns 0..C-1 from the attention
output, and linear2 is one block-scaled FP8 GEMM with K = 5C.  The model hands the quantized weights and workspaces to the
processors on `vec` (`_osb_fp8`, an `Fp8State`).

FP8 attention (MMDiTModel.enable_fp8_attention, independent of the FP8 MLPs): the joint self-attention runs on
`osb_attn_fp8` (q / k quantized per token and head after QK-norm and RoPE, v per channel, P as e4m3(256 p)) instead of
`osb_attn_short`, with the workspaces on `vec` (`_osb_fp8_attn`, an `Fp8AttnState`).  No Linear changes.

FP8 projections (MMDiTModel.enable_fp8(projections=True), `Fp8State.proj`): every block Linear runs on e4m3.  Double
blocks, per stream: ln_modulate_fp8 -> the q|k|v GEMM on per-row A (`osb_gemm_fp8_blocks`, bf16 out) -> attention whose
output leaves as e4m3 codes with 1 x 128 block scales (`osb_attn_fp8_blocks` with FP8 attention on, else the bf16
attention and `osb_quant_blocks_fp8`) -> `proj` on block-scaled A (gate + residual).  Single blocks: ONE ln_modulate_fp8
pass feeds the qkv GEMM and the mlp GEMM, the attention output fills columns 0..C-1 of the e4m3 cat buffer the same
way, and no bf16 LN pass runs.

LoRA on FP8 (MMDiTModel.enable_fp8(..., lora=True), `Fp8State.lora`): an adapter on a Linear that runs on e4m3 is applied by
`osb_gemm_fp8_lora` (the FP8 GEMM with U (s B)^T, and DoRA's column scale, in the same fp32 accumulator).  Its down
projection U = x A_cat^T reads the e4m3 codes the base GEMM reads (per-row codes of ln_modulate_fp8 for q|k|v, fc1 and
linear1; block-scaled codes for proj, fc2 and linear2) on `osb_gemm_fp8_blocks` with A_cat quantized per row, one down
GEMM per shared input as on the bf16 path."""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch
from torch import Tensor, nn

from opensora.utils.lora import adapter_of, lora_pack

from .math import liger_rope, rope, rope_tables


def _osb():
    import osb200

    return osb200


class EmbedND(nn.Module):
    """layers.py:31-44."""

    def __init__(self, dim: int, theta: int, axes_dim: list[int]):
        super().__init__()
        self.dim, self.theta, self.axes_dim = dim, theta, axes_dim

    def forward(self, ids: Tensor) -> Tensor:
        emb = torch.cat([rope(ids[..., i], self.axes_dim[i], self.theta) for i in range(ids.shape[-1])], dim=-3)
        return emb.unsqueeze(1)


class LigerEmbedND(nn.Module):
    """layers.py:47-65."""

    def __init__(self, dim: int, theta: int, axes_dim: list[int]):
        super().__init__()
        self.dim, self.theta, self.axes_dim = dim, theta, axes_dim

    def forward(self, ids: Tensor):
        cs = [liger_rope(ids[..., i], self.axes_dim[i], self.theta) for i in range(ids.shape[-1])]
        cos = torch.cat([c for c, _ in cs], dim=-1).repeat(1, 1, 2).contiguous()
        sin = torch.cat([s for _, s in cs], dim=-1).repeat(1, 1, 2).contiguous()
        return (cos, sin)


def timestep_embedding(t: Tensor, dim, max_period=10000, time_factor: float = 1000.0):
    """layers.py:68-88 (the reference `torch.compile`s this; it is [B, 256] work once per step)."""
    t = time_factor * t
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(0, half, dtype=torch.float32) / half).to(t.device)
    args = t[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    if torch.is_floating_point(t):
        emb = emb.to(t)
    return emb


def linear_parts(lin: nn.Module, k_pad: int = 0):
    """(weight, bias, lora) of a Linear the forward sends to osb200: lora is None, or (A [r, K + k_pad], scaling * B,
    DoRA column scale or None) of its adapter (lora_pack)."""
    if adapter_of(lin) is None:
        return lin.weight, lin.bias, None
    A, (B,), (S,) = lora_pack([[(lin, 0, lin.out_features)]], k_pad)
    return lin.weight, lin.bias, (A, B, S)


def _gemm(osb, x2d: Tensor, w: Tensor, b, lora, u: Tensor | None = None, **kw) -> Tensor:
    """osb.gemm, or with lora = (A, B, col_scale) the fused base + update GEMM; `u` = x2d A^T when a shared down GEMM
    made it."""
    if lora is None or lora[1] is None:
        return osb.gemm(x2d, w, b, **kw)
    if u is None:
        u = osb.gemm(x2d, lora[0])
    if lora[2] is not None:
        kw["col_scale"] = lora[2]
    return osb.gemm_lora(x2d, w, b, u, lora[1], **kw)


def _gemm8(osb, a8: Tensor, a_s: Tensor, w8: Tensor, w_s: Tensor, b, lora, u: Tensor | None, **kw):
    """osb.gemm_fp8_blocks, or with lora = (A_cat, B, col_scale) and its down projection `u` the FP8 GEMM with the
    unmerged update (osb.gemm_fp8_lora)."""
    if lora is None or lora[1] is None:
        return osb.gemm_fp8_blocks(a8, a_s, w8, w_s, b, **kw)
    return osb.gemm_fp8_lora(a8, a_s, w8, w_s, b, u, lora[1], col_scale=lora[2], **kw)


def _one(pack, i: int = 0):
    """(A_cat, B, col_scale) of group i of a lora_pack result, or None."""
    return None if pack is None else (pack[0], pack[1][i], pack[2][i])


def _linear(x2d: Tensor, lin: nn.Linear, **kw) -> Tensor:
    return _gemm(_osb(), x2d, *linear_parts(lin), **kw)


class MLPEmbedder(nn.Module):
    def __init__(self, in_dim: int, hidden_dim: int):
        super().__init__()
        self.in_layer = nn.Linear(in_dim, hidden_dim, bias=True)
        self.silu = nn.SiLU()
        self.out_layer = nn.Linear(hidden_dim, hidden_dim, bias=True)

    def forward(self, x: Tensor) -> Tensor:
        h = _linear(x.to(self.in_layer.weight.dtype).contiguous(), self.in_layer)
        return _linear(torch.nn.functional.silu(h), self.out_layer)


class RMSNorm(nn.Module):
    """Parameter container (`scale`), layers.py:102-111; applied inside the attention kernel."""

    def __init__(self, dim: int):
        super().__init__()
        self.scale = nn.Parameter(torch.ones(dim))


class FusedRMSNorm(RMSNorm):
    pass


class QKNorm(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.query_norm = FusedRMSNorm(dim)
        self.key_norm = FusedRMSNorm(dim)


class SelfAttention(nn.Module):
    """Parameter container with the reference's attribute names (layers.py:138-152)."""

    def __init__(self, dim: int, num_heads: int = 8, qkv_bias: bool = False, fused_qkv: bool = True):
        super().__init__()
        self.num_heads, self.fused_qkv = num_heads, fused_qkv
        if fused_qkv:
            self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        else:
            self.q_proj = nn.Linear(dim, dim, bias=qkv_bias)
            self.k_proj = nn.Linear(dim, dim, bias=qkv_bias)
            self.v_proj = nn.Linear(dim, dim, bias=qkv_bias)
        self.norm = QKNorm(dim // num_heads)
        self.proj = nn.Linear(dim, dim)


@dataclass
class ModulationOut:
    shift: Tensor
    scale: Tensor
    gate: Tensor


class Modulation(nn.Module):
    """Parameter container (layers.py:179-192); the processors read `lin` / `multiplier` and run the projection on
    osb200.  `forward` keeps the reference's return contract for callers outside the block path."""

    def __init__(self, dim: int, double: bool):
        super().__init__()
        self.is_double = double
        self.multiplier = 6 if double else 3
        self.lin = nn.Linear(dim, self.multiplier * dim, bias=True)

    def forward(self, vec: Tensor):
        out = _linear(torch.nn.functional.silu(vec).contiguous(), self.lin)[:, None, :].chunk(self.multiplier, dim=-1)
        return ModulationOut(*out[:3]), (ModulationOut(*out[3:]) if self.is_double else None)


def _check(x: Tensor):
    osb = _osb()
    osb.require_cuda_bf16(x, "MMDiT")
    return osb


def _rope(pe):
    """(cos, sin, rotate_half) for the attention kernel: EmbedND -> interleaved pairs, LigerEmbedND -> rotate-half.  The
    tables depend only on `pe`, which every block of a forward (and, with a cached `pe`, every step) shares: they are memoised on
    the tensor itself (57 slicing + contiguous passes per step otherwise)."""
    host = pe if isinstance(pe, Tensor) else pe[0]
    hit = getattr(host, "_osb_rope_tables", None)
    if hit is None or hit[0] != host._version:
        hit = (host._version, rope_tables(pe))
        try:
            host._osb_rope_tables = hit
        except Exception:   # a tensor subclass that refuses attributes: just recompute
            pass
    return hit[1]


# Sequence parallelism (Ulysses, the reference's `all_to_all` mode: opensora/models/mmdit/distributed.py:473-495): the joint
# txt|img sequence is split into P equal chunks; around attention q, k, v are exchanged "scatter heads / gather sequence" and
# the output back.  MMDiTModel sets the group for the duration of a forward; a processor running outside of it sees None.
_SP = {"group": None}


def _sp_group():
    return _SP["group"]


class Fp8AttnState:
    """What the FP8 attention path of one MMDiTModel keeps: the workspaces of `osb200.attn_fp8`, one per (B, L, heads,
    device), reused by every block."""

    def __init__(self):
        self._ws = {}

    def workspace(self, osb, B: int, L: int, H: int, device):
        key = (B, L, H, device)
        ws = self._ws.get(key)
        if ws is None:
            ws = self._ws[key] = osb.attn_fp8_workspace(B, L, H, device)
        return ws


def _attention(osb, fp8_attn: Fp8AttnState | None, q, k, v, out, B: int, L: int, H: int, D: int, norm_split: int,
               attn_kw: dict, out_scale: Tensor | None = None) -> None:
    """Joint self-attention of B sequences of L tokens: `osb_attn_short`, or `osb_attn_fp8` when FP8 attention is on
    (`osb_attn_fp8_blocks` with `out_scale`: e4m3 `out`, one scale per (token, head))."""
    kw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H,
              head_dim=D, norm_split=norm_split, **attn_kw)
    if fp8_attn is None:
        osb.attn_short(q, k, v, out, **kw)
    elif out_scale is not None:
        osb.attn_fp8_blocks(q, k, v, out, out_scale, workspace=fp8_attn.workspace(osb, B, L, H, q.device), **kw)
    else:
        osb.attn_fp8(q, k, v, out, workspace=fp8_attn.workspace(osb, B, L, H, q.device), **kw)


def _attention_e4m3(osb, fp8_attn: Fp8AttnState | None, q, k, v, out8, B: int, L: int, H: int, D: int,
                    norm_split: int, attn_kw: dict) -> None:
    """`_attention` written as e4m3 codes with 1 x 128 block scales into out8 = (codes [rows, H*D], scales
    [rows, H*D / 128]): by the FP8 attention kernel itself, or after the bf16 attention by `osb_quant_blocks_fp8`."""
    if fp8_attn is not None:
        _attention(osb, fp8_attn, q, k, v, out8[0], B, L, H, D, norm_split, attn_kw, out_scale=out8[1])
        return
    ao = torch.empty(B * L, H * D, dtype=q.dtype, device=q.device)
    _attention(osb, None, q, k, v, ao, B, L, H, D, norm_split, attn_kw)
    osb.quant_blocks_fp8(ao, out=out8[0], out_scale=out8[1])


def _sp_attention(osb, qkv: Tensor, out_cols: int, B: int, Lloc: int, H: int, D: int, attn_kw: dict, norm_split_full: int,
                  dtype, device, fp8_attn: Fp8AttnState | None = None, out8=None) -> Tensor | None:
    """softmax(q k^T) v over the FULL joint sequence from this rank's [B*Lloc, 3*H*D] q|k|v rows: heads are scattered and
    the sequence gathered with one all-to-all (q, k, v travel together), attention runs on H/P heads, and the output comes
    back with the inverse exchange.  Without a group it is the plain local attention.  With `fp8_attn` the attention
    itself runs on FP8 operands (it sees the whole sequence of its heads either way).
    With out8 = (codes, scales) the output is written there as e4m3 with 1 x 128 block scales (`_attention_e4m3`) and
    None is returned; the inverse exchange then carries the codes (as bytes) and the per-(token, head) scales of the FP8
    attention, or the bf16 rows that are quantized after it.  A (token, head) block is quantized alone either way, so
    the codes equal the single-rank ones."""
    import torch.distributed as dist

    from opensora.acceleration.communications import all_to_all

    g = _sp_group()
    P = dist.get_world_size(g) if g is not None else 1
    C = H * D
    if P == 1 and out8 is not None:
        _attention_e4m3(osb, fp8_attn, qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out8, B, Lloc, H, D, norm_split_full,
                        attn_kw)
        return None
    if P == 1:
        ao = torch.empty(B * Lloc, out_cols, dtype=dtype, device=device)
        _attention(osb, fp8_attn, qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], ao[:, :C], B, Lloc, H, D,
                   norm_split_full, attn_kw)
        return ao
    if H % P:
        raise ValueError(f"sequence parallel size {P} must divide the head count {H} (distributed.py:477-479)")
    Hp, L = H // P, Lloc * P
    full = all_to_all(qkv.view(B, Lloc, 3, H, D), g, scatter_dim=3, gather_dim=1).reshape(B * L, 3 * Hp * D)
    Cp = Hp * D
    if out8 is not None and fp8_attn is not None:
        c8 = torch.empty(B * L, Cp, dtype=torch.float8_e4m3fn, device=device)
        s8 = torch.empty(B * L, Hp, dtype=torch.float32, device=device)
        _attention(osb, fp8_attn, full[:, :Cp], full[:, Cp:2 * Cp], full[:, 2 * Cp:], c8, B, L, Hp, D, norm_split_full,
                   attn_kw, out_scale=s8)
        back8 = all_to_all(c8.view(torch.uint8).view(B, L, Hp, D), g, scatter_dim=1, gather_dim=2)
        out8[0].copy_(back8.view(torch.float8_e4m3fn).reshape(B * Lloc, C))
        out8[1].copy_(all_to_all(s8.view(B, L, Hp), g, scatter_dim=1, gather_dim=2).reshape(B * Lloc, H))
        return None
    ao_full = torch.empty(B * L, Cp, dtype=dtype, device=device)
    _attention(osb, fp8_attn, full[:, :Cp], full[:, Cp:2 * Cp], full[:, 2 * Cp:], ao_full, B, L, Hp, D, norm_split_full,
               attn_kw)
    back = all_to_all(ao_full.view(B, L, Hp, D), g, scatter_dim=1, gather_dim=2).reshape(B * Lloc, C)
    if out8 is not None:
        osb.quant_blocks_fp8(back, out=out8[0], out_scale=out8[1])
        return None
    if out_cols == C:
        return back
    ao = torch.empty(B * Lloc, out_cols, dtype=dtype, device=device)
    ao[:, :C] = back
    return ao


class Fp8State:
    """What the FP8 path of one MMDiTModel keeps: e4m3 weights with per-output-channel scales, quantized once per block
    and MLP (`weights`) and, with `proj`, per block and stream for the q|k|v and attention-output projections
    (`proj_weights`), and e4m3 / scale workspaces reused by every block, one per shape (`buf`).  With `lora`, adapters on
    those Linears run on the FP8 path: the e4m3 copy of each pack's A_cat is cached per use (`down`)."""

    def __init__(self, proj: bool = False, lora: bool = False):
        self.proj, self.lora = proj, lora
        self._w, self._ws, self._la = {}, {}, {}

    @staticmethod
    def proj_linears(blk: nn.Module, kind: str):
        """The Linears holding the projections of the FP8 projection path: the q|k|v Linears and `proj` of one stream
        (kind "img" / "txt"), or linear1 (q_proj, k_proj, v_mlp) of a single block, which hold its q|k|v rows."""
        if kind != "single":
            sa = blk.img_attn if kind == "img" else blk.txt_attn
            qkv = (sa.qkv,) if getattr(sa, "fused_qkv", hasattr(sa, "qkv")) else (sa.q_proj, sa.k_proj, sa.v_proj)
            return qkv + (sa.proj,)
        if getattr(blk, "fused_qkv", hasattr(blk, "linear1")):
            return (blk.linear1,)
        return (blk.q_proj, blk.k_proj, blk.v_mlp)

    def proj_weights(self, osb, blk: nn.Module, kind: str):
        """(q|k|v e4m3 [3C, C], scales [3C], bias or None, proj e4m3 [C, C], scales [C], bias) of one stream of a double
        block; the last three are None for a single block.  q|k|v rows in the order of the bf16 path's packing."""
        key = (id(blk), kind, "proj")
        hit = self._w.get(key)
        if hit is None or hit[0] is not blk:
            lins = self.proj_linears(blk, kind)
            for lin in lins:
                if adapter_of(lin) is not None and not self.lora:
                    raise ValueError("FP8 projections: a LoRA / DoRA adapter on a projection Linear cannot run on the FP8 "
                                     "path; unload_lora or disable_fp8 first")
            if kind != "single":
                qkv, proj = lins[:-1], lins[-1]
                C = proj.out_features
                w = qkv[0].weight if len(qkv) == 1 else torch.cat([lin.weight for lin in qkv], 0)
                b = None if qkv[0].bias is None else (
                    qkv[0].bias if len(qkv) == 1 else torch.cat([lin.bias for lin in qkv], 0).contiguous())
            else:
                C = blk.linear2.out_features
                if len(lins) == 1:
                    w, b = lins[0].weight[:3 * C], lins[0].bias[:3 * C]
                else:
                    w = torch.cat([lins[0].weight, lins[1].weight, lins[2].weight[:C]], 0)
                    b = torch.cat([lins[0].bias, lins[1].bias, lins[2].bias[:C]], 0).contiguous()
                proj = None
            wq, sq = osb.quant_blocks_fp8(w, block=C)
            pw = (None, None, None)
            if proj is not None:
                wp, sp = osb.quant_blocks_fp8(proj.weight, block=C)
                pw = (wp, sp.view(-1), proj.bias)
            hit = self._w[key] = (blk, (wq, sq.view(-1), b) + pw)
        return hit[1]

    @staticmethod
    def mlp_linears(blk: nn.Module, kind: str):
        """(fc1-side Linear, its row range, fc2-side Linear) of an MLP: kind "img" / "txt" (double block) or "single"."""
        if kind != "single":
            mlp = blk.img_mlp if kind == "img" else blk.txt_mlp
            return mlp[0], (0, mlp[0].out_features), mlp[2]
        C = blk.linear2.out_features
        lin1 = blk.linear1 if getattr(blk, "fused_qkv", hasattr(blk, "linear1")) else blk.v_mlp
        off = 3 * C if lin1 is getattr(blk, "linear1", None) else C
        return lin1, (off, lin1.out_features), blk.linear2

    def weights(self, osb, blk: nn.Module, kind: str):
        """(fc1 e4m3 [hid, C], fc1 scales [hid], fc1 bias, fc2 e4m3 [C, K2], fc2 scales [C], fc2 bias) of one MLP."""
        key = (id(blk), kind)
        hit = self._w.get(key)
        if hit is None or hit[0] is not blk:
            l1, (lo, hi), l2 = self.mlp_linears(blk, kind)
            for lin in (l1, l2):
                if adapter_of(lin) is not None and not self.lora:
                    raise ValueError("FP8 MLPs: a LoRA / DoRA adapter on an MLP Linear cannot run on the FP8 path; "
                                     "unload_lora or disable_fp8 first")
            w1, s1 = osb.quant_blocks_fp8(l1.weight[lo:hi], block=l1.in_features)
            w2, s2 = osb.quant_blocks_fp8(l2.weight, block=l2.in_features)
            b1 = None if l1.bias is None else l1.bias[lo:hi]
            hit = self._w[key] = (blk, (w1, s1.view(-1), b1, w2, s2.view(-1), l2.bias))
        return hit[1]

    def pack(self, groups):
        """lora_pack(groups) when adapters run on the FP8 path, else None."""
        return lora_pack(groups) if self.lora else None

    def mlp_lora(self, blk: nn.Module, kind: str):
        """(fc1 adapter, fc2 adapter) of one MLP as (A_cat, B, col_scale) or None each (see mlp_linears)."""
        if not self.lora:
            return None, None
        l1, (lo, hi), l2 = self.mlp_linears(blk, kind)
        return _one(lora_pack([[(l1, lo, hi)]])), _one(lora_pack([[(l2, 0, l2.out_features)]]))

    def down(self, osb, key, lora, a8: Tensor, a_s: Tensor) -> Tensor | None:
        """U = x A_cat^T (bf16 [rows, R]) of the adapters whose GEMMs read the e4m3 input (a8, a_s), on the block-scaled
        FP8 GEMM; `lora` is a pack or one of its groups (A_cat first), None without adapters.  A_cat is quantized per row once per `key` and pack: lora_pack hands out a new
        A_cat whenever the adapter state changes (reload, edited A / B, DoRA magnitude or base weight)."""
        if lora is None:
            return None
        A = lora[0]
        hit = self._la.get(key)
        if hit is None or hit[0] is not A:
            q, sc = osb.quant_blocks_fp8(A, block=A.shape[1])
            hit = self._la[key] = (A, q, sc.view(-1))
        return osb.gemm_fp8_blocks(a8, a_s, hit[1], hit[2])

    def buf(self, name: str, *shape, dtype=torch.float32, device=None) -> Tensor:
        key = (name, shape, dtype, device)
        t = self._ws.get(key)
        if t is None:
            t = self._ws[key] = torch.empty(shape, dtype=dtype, device=device)
        return t


def _mlp_fp8(osb, fp8: Fp8State, blk: nn.Module, kind: str, x: Tensor, mod, n: int) -> None:
    """x += gate * MLP((1 + scale) * LN(x) + shift) in place, on FP8 operands (x: [rows, C] bf16, group_rows = n)."""
    w1, s1, b1, w2, s2, b2 = fp8.weights(osb, blk, kind)
    l1, l2 = fp8.mlp_lora(blk, kind)
    rows, C = x.shape
    hid, dev, f8 = w1.shape[0], x.device, torch.float8_e4m3fn
    x8, xs = osb.ln_modulate_fp8(x, mod.shift, mod.scale, group_rows=n, out=fp8.buf("x8", rows, C, dtype=f8, device=dev),
                                 out_scale=fp8.buf("xs", rows, device=dev))
    h8, hs = _gemm8(osb, x8, xs, w1, s1, b1, l1, fp8.down(osb, (id(blk), kind, "fc1"), l1, x8, xs),
                    epilogue=osb.EPI_BIAS_GELU_TANH_FP8, out=fp8.buf("h8", rows, hid, dtype=f8, device=dev),
                    out_scale=fp8.buf("hs", rows, hid // 128, device=dev))
    _gemm8(osb, h8, hs, w2, s2, b2, l2, fp8.down(osb, (id(blk), kind, "fc2"), l2, h8, hs), epilogue=osb.EPI_BIAS_GATE_RES,
           residual=x, gate=mod.gate, group_rows=n, out=x)


def _qkv_fp8(osb, fp8: Fp8State, blk: nn.Module, kind: str, x: Tensor, mod, n: int, qkv: Tensor, L: int,
             off: int) -> tuple[Tensor, Tensor]:
    """q|k|v = W_qkv ((1 + scale) * LN(x) + shift) + b on FP8 operands: one ln_modulate_fp8 pass (codes + row scales,
    returned) and, per sample of n rows, one row-scaled e4m3 GEMM into rows b*L + off .. of the joint buffer `qkv`."""
    wq, sq, bq = fp8.proj_weights(osb, blk, kind)[:3]
    lq = _ProcessorBase._qkv_lora(blk.img_attn if kind == "img" else blk.txt_attn) if fp8.lora else None
    rows, C = x.shape
    dev, f8 = x.device, torch.float8_e4m3fn
    x8, xs = osb.ln_modulate_fp8(x, mod.shift, mod.scale, group_rows=n, out=fp8.buf("x8", rows, C, dtype=f8, device=dev),
                                 out_scale=fp8.buf("xs", rows, device=dev))
    u = fp8.down(osb, (id(blk), kind, "qkv"), lq, x8, xs)   # one down projection over all rows of the stream
    for b in range(rows // n):
        r = slice(b * n, (b + 1) * n)
        _gemm8(osb, x8[r], xs[r], wq, sq, bq, lq, None if u is None else u[r], out=qkv[b * L + off:b * L + off + n])
    return x8, xs


class _ProcessorBase:
    """What both processors share.  A processor holds NO model weights and touches only attributes the reference's own
    block classes have (`opensora/models/mmdit/layers.py:138-176,256-306,337-388`), so it can be installed with
    `block.set_processor(...)` on the reference's DoubleStreamBlock / SingleStreamBlock objects as well as on this
    package's.  Derived tensors (q|k|v weights concatenated for checkpoints with `fused_qkv=False`) are cached per
    block, keyed by the identity and version of the source parameters, so `.to()` / `load_state_dict` invalidate them."""

    def __init__(self):
        import weakref

        self._cache = weakref.WeakKeyDictionary()

    def _cached(self, block: nn.Module, name: str, sources, build):
        sig = tuple((t.data_ptr(), t._version, t.dtype, t.device) for t in sources if t is not None)
        ent = self._cache.setdefault(block, {})
        hit = ent.get(name)
        if hit is None or hit[0] != sig:
            ent[name] = hit = (sig, build())
        return hit[1]

    def _qkv(self, block: nn.Module, sa: nn.Module, name: str):
        """[3C, C] weight and [3C] bias in q|k|v row order for ONE GEMM, whichever way the checkpoint stores them."""
        if getattr(sa, "fused_qkv", hasattr(sa, "qkv")):
            return sa.qkv.weight, sa.qkv.bias
        ws = (sa.q_proj.weight, sa.k_proj.weight, sa.v_proj.weight)
        bs = (sa.q_proj.bias, sa.k_proj.bias, sa.v_proj.bias)
        return self._cached(block, name, ws + bs, lambda: (
            torch.cat(ws, 0).contiguous(), None if bs[0] is None else torch.cat(bs, 0).contiguous()))

    @staticmethod
    def _qkv_lora(sa: nn.Module):
        """Adapters of the q|k|v projection in the row order of `_qkv`: (A_cat, B_cat, col_scale) or None."""
        if getattr(sa, "fused_qkv", hasattr(sa, "qkv")):
            return linear_parts(sa.qkv)[2]
        C = sa.q_proj.out_features
        p = lora_pack([[(sa.q_proj, 0, C), (sa.k_proj, 0, C), (sa.v_proj, 0, C)]])
        return None if p is None else (p[0], p[1][0], p[2][0])

    @staticmethod
    def _modulation(osb, mod: nn.Module, vec: Tensor):
        """layers.py:186-192 on osb200: lin(silu(vec)) -> fp32 [B, C] row views (row stride multiplier*C) the kernels take
        as shift / scale / gate.  When the model has already projected `vec` through EVERY block's modulation layer in one
        grouped GEMM (MMDiTModel.forward_ckpt: SURVEY.md 8f-2), the result rides on `vec` and this block takes its columns."""
        grouped = getattr(vec, "_osb_grouped_modulation", None)
        if grouped is not None and id(mod.lin) in grouped[1]:
            lo, hi = grouped[1][id(mod.lin)]
            out = grouped[0][:, lo:hi]
        else:
            out = _gemm(osb, torch.nn.functional.silu(vec).contiguous(), *linear_parts(mod.lin)).float()
        mult = getattr(mod, "multiplier", None) or (mod.lin.out_features // mod.lin.in_features)
        c = out.chunk(mult, dim=-1)
        return ModulationOut(*c[:3]), (ModulationOut(*c[3:6]) if mult >= 6 else None)


class DoubleStreamBlockProcessor(_ProcessorBase):
    """osb200 implementation of layers.py:195-253 (and, under sequence parallelism, of distributed.py:473-495)."""

    def __call__(self, attn: nn.Module, img: Tensor, txt: Tensor, vec: Tensor, pe) -> tuple[Tensor, Tensor]:
        osb = _check(img)
        B, Li, C = img.shape
        Lt = txt.shape[1]            # may be 0 on a sequence-parallel rank whose chunk holds image tokens only
        L, H = Lt + Li, attn.num_heads
        D = C // H
        im1, im2 = self._modulation(osb, attn.img_mod, vec)
        tm1, tm2 = self._modulation(osb, attn.txt_mod, vec)
        img2, txt2 = img.reshape(B * Li, C).contiguous(), txt.reshape(B * Lt, C).contiguous()
        # q|k|v of both streams land in ONE joint [B*(Lt+Li), 3C] buffer in txt-then-img token order (layers.py:240-242)
        qkv = torch.empty(B * L, 3 * C, dtype=img.dtype, device=img.device)
        fp8 = getattr(vec, "_osb_fp8", None)
        proj8 = fp8 is not None and fp8.proj
        if proj8:
            for x2, mod, n, off, kind in ((img2, im1, Li, Lt, "img"), (txt2, tm1, Lt, 0, "txt")):
                if n:
                    _qkv_fp8(osb, fp8, attn, kind, x2, mod, n, qkv, L, off)
        else:
            self._qkv_bf16(osb, attn, img2, txt2, im1, tm1, qkv, B, Li, Lt)
        cos, sin, half = _rope(pe)
        kw = dict(q_norm_w=attn.txt_attn.norm.query_norm.scale, k_norm_w=attn.txt_attn.norm.key_norm.scale,
                  q_norm_w2=attn.img_attn.norm.query_norm.scale, k_norm_w2=attn.img_attn.norm.key_norm.scale,
                  rope_cos=cos, rope_sin=sin, rope_half=half)
        # tokens at joint position >= the FULL text length take the image stream's QK-norm weights
        split_full = getattr(vec, "_osb_txt_len", Lt)
        img_o, txt_o = torch.empty_like(img2), torch.empty_like(txt2)
        if proj8:   # attention output as e4m3 + 1 x 128 block scales -> x + gate * proj(attn) on FP8 operands
            rows, f8, dev = B * L, torch.float8_e4m3fn, img.device
            ao8 = (fp8.buf("ao8", rows, C, dtype=f8, device=dev), fp8.buf("aos", rows, C // 128, device=dev))
            _sp_attention(osb, qkv, C, B, L, H, D, kw, split_full, img.dtype, dev, getattr(vec, "_osb_fp8_attn", None),
                          out8=ao8)
            # both output projections read ao8: one down projection for their adapters
            lp = fp8.pack([[(attn.img_attn.proj, 0, C)], [(attn.txt_attn.proj, 0, C)]])
            up = fp8.down(osb, (id(attn), "proj"), lp, ao8[0], ao8[1])
            for i, (x2, x_o, mod, n, off, kind) in enumerate(((img2, img_o, im1, Li, Lt, "img"),
                                                              (txt2, txt_o, tm1, Lt, 0, "txt"))):
                wp, sp, bp = fp8.proj_weights(osb, attn, kind)[3:]
                for b in range(B if n else 0):
                    r = slice(b * L + off, b * L + off + n)
                    _gemm8(osb, ao8[0][r], ao8[1][r], wp, sp, bp, _one(lp, i), None if up is None else up[r],
                           epilogue=osb.EPI_BIAS_GATE_RES, residual=x2[b * n:(b + 1) * n], gate=mod.gate[b:b + 1],
                           out=x_o[b * n:(b + 1) * n])
        else:
            self._proj_bf16(osb, attn, qkv, kw, split_full, img2, txt2, img_o, txt_o, im1, tm1, vec, B, L, Li, Lt, H, D)
        # x + gate * MLP((1 + scale) * LN(x) + shift)   (layers.py:248, 252)
        for x_o, mod, mlp, n, kind in ((img_o, im2, attn.img_mlp, Li, "img"), (txt_o, tm2, attn.txt_mlp, Lt, "txt")):
            if n == 0:
                continue
            if fp8 is not None:
                _mlp_fp8(osb, fp8, attn, kind, x_o, mod, n)
                continue
            xm = osb.ln_modulate(x_o, mod.shift, mod.scale, group_rows=n)
            hid = _gemm(osb, xm, *linear_parts(mlp[0]), epilogue=osb.EPI_BIAS_GELU_TANH)
            _gemm(osb, hid, *linear_parts(mlp[2]), epilogue=osb.EPI_BIAS_GATE_RES, residual=x_o, gate=mod.gate,
                  group_rows=n, out=x_o)
        return img_o.view(B, Li, C), txt_o.view(B, Lt, C)

    def _qkv_bf16(self, osb, attn, img2, txt2, im1, tm1, qkv, B, Li, Lt):
        """q|k|v of both streams on bf16 GEMMs (with their adapters) into the joint buffer."""
        L = Lt + Li
        wi, bi = self._qkv(attn, attn.img_attn, "img_qkv")
        wt, bt = self._qkv(attn, attn.txt_attn, "txt_qkv")
        li, lt = self._qkv_lora(attn.img_attn), self._qkv_lora(attn.txt_attn)
        ui = ut = None   # adapters: one down projection over all rows of a stream, sliced per sample below
        if Li:
            xi = osb.ln_modulate(img2, im1.shift, im1.scale, group_rows=Li)
            ui = None if li is None else osb.gemm(xi, li[0])
        if Lt:
            xt = osb.ln_modulate(txt2, tm1.shift, tm1.scale, group_rows=Lt)
            ut = None if lt is None else osb.gemm(xt, lt[0])
        for b in range(B):
            if Lt:
                _gemm(osb, xt[b * Lt:(b + 1) * Lt], wt, bt, lt, None if ut is None else ut[b * Lt:(b + 1) * Lt],
                      out=qkv[b * L:b * L + Lt])
            if Li:
                _gemm(osb, xi[b * Li:(b + 1) * Li], wi, bi, li, None if ui is None else ui[b * Li:(b + 1) * Li],
                      out=qkv[b * L + Lt:(b + 1) * L])

    @staticmethod
    def _proj_bf16(osb, attn, qkv, kw, split_full, img2, txt2, img_o, txt_o, im1, tm1, vec, B, L, Li, Lt, H, D):
        """Attention in bf16 out and x + gate * proj(attn) of both streams on bf16 GEMMs (with their adapters)."""
        C = img2.shape[1]
        ao = _sp_attention(osb, qkv, C, B, L, H, D, kw, split_full, img2.dtype, img2.device,
                           getattr(vec, "_osb_fp8_attn", None))
        # both output projections read `ao`: one down projection for their adapters
        pi, pt = attn.img_attn.proj, attn.txt_attn.proj
        lp = lora_pack([[(pi, 0, pi.out_features)], [(pt, 0, pt.out_features)]])
        up = None if lp is None else osb.gemm(ao, lp[0])
        lpi, lpt = (None, None) if lp is None else ((lp[0], lp[1][0], lp[2][0]), (lp[0], lp[1][1], lp[2][1]))
        for b in range(B):  # x + gate * proj(attn)   (layers.py:247, 251)
            if Li:
                _gemm(osb, ao[b * L + Lt:(b + 1) * L], pi.weight, pi.bias, lpi,
                      None if up is None else up[b * L + Lt:(b + 1) * L],
                      epilogue=osb.EPI_BIAS_GATE_RES, residual=img2[b * Li:(b + 1) * Li], gate=im1.gate[b:b + 1],
                      out=img_o[b * Li:(b + 1) * Li])
            if Lt:
                _gemm(osb, ao[b * L:b * L + Lt], pt.weight, pt.bias, lpt, None if up is None else up[b * L:b * L + Lt],
                      epilogue=osb.EPI_BIAS_GATE_RES, residual=txt2[b * Lt:(b + 1) * Lt], gate=tm1.gate[b:b + 1],
                      out=txt_o[b * Lt:(b + 1) * Lt])


class DoubleStreamBlock(nn.Module):
    def __init__(self, hidden_size: int, num_heads: int, mlp_ratio: float, qkv_bias: bool = False, fused_qkv: bool = True):
        super().__init__()
        mlp_hidden_dim = int(hidden_size * mlp_ratio)
        self.num_heads, self.hidden_size, self.head_dim = num_heads, hidden_size, hidden_size // num_heads
        self.img_mod = Modulation(hidden_size, double=True)
        self.img_norm1 = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.img_attn = SelfAttention(dim=hidden_size, num_heads=num_heads, qkv_bias=qkv_bias, fused_qkv=fused_qkv)
        self.img_norm2 = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.img_mlp = nn.Sequential(nn.Linear(hidden_size, mlp_hidden_dim, bias=True), nn.GELU(approximate="tanh"),
                                     nn.Linear(mlp_hidden_dim, hidden_size, bias=True))
        self.txt_mod = Modulation(hidden_size, double=True)
        self.txt_norm1 = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.txt_attn = SelfAttention(dim=hidden_size, num_heads=num_heads, qkv_bias=qkv_bias, fused_qkv=fused_qkv)
        self.txt_norm2 = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.txt_mlp = nn.Sequential(nn.Linear(hidden_size, mlp_hidden_dim, bias=True), nn.GELU(approximate="tanh"),
                                     nn.Linear(mlp_hidden_dim, hidden_size, bias=True))
        self.set_processor(DoubleStreamBlockProcessor())

    def set_processor(self, processor) -> None:
        self.processor = processor

    def get_processor(self):
        return self.processor

    def forward(self, img: Tensor, txt: Tensor, vec: Tensor, pe, **kwargs) -> tuple[Tensor, Tensor]:
        return self.processor(self, img, txt, vec, pe)


class SingleStreamBlockProcessor(_ProcessorBase):
    """osb200 implementation of layers.py:309-334."""

    def _split_weights(self, blk: nn.Module):
        """(W_qkv [3C,C], b_qkv, W_mlp [4C,C], b_mlp): row views of linear1, or packed from q_proj / k_proj / v_mlp."""
        C = blk.linear2.out_features
        if getattr(blk, "fused_qkv", hasattr(blk, "linear1")):
            w, b = blk.linear1.weight, blk.linear1.bias
            return w[:3 * C], b[:3 * C], w[3 * C:], b[3 * C:]
        src = (blk.q_proj.weight, blk.k_proj.weight, blk.v_mlp.weight, blk.q_proj.bias, blk.k_proj.bias, blk.v_mlp.bias)
        wq, bq = self._cached(blk, "qkv", src, lambda: (
            torch.cat([blk.q_proj.weight, blk.k_proj.weight, blk.v_mlp.weight[:C]], 0).contiguous(),
            torch.cat([blk.q_proj.bias, blk.k_proj.bias, blk.v_mlp.bias[:C]], 0).contiguous()))
        return wq, bq, blk.v_mlp.weight[C:], blk.v_mlp.bias[C:]

    @staticmethod
    def _split_lora(blk: nn.Module, M4: int):
        """Adapters of the qkv and mlp parts of `_split_weights`, which read the same input: ((A_cat, B_qkv, S_qkv),
        (A_cat, B_mlp, S_mlp)) with one A_cat for both, or None."""
        C = blk.linear2.out_features
        if getattr(blk, "fused_qkv", hasattr(blk, "linear1")):
            groups = [[(blk.linear1, 0, 3 * C)], [(blk.linear1, 3 * C, 3 * C + M4)]]
        else:
            groups = [[(blk.q_proj, 0, C), (blk.k_proj, 0, C), (blk.v_mlp, 0, C)], [(blk.v_mlp, C, C + M4)]]
        p = lora_pack(groups)
        return None if p is None else ((p[0], p[1][0], p[2][0]), (p[0], p[1][1], p[2][1]))

    def __call__(self, attn: nn.Module, x: Tensor, vec: Tensor, pe) -> Tensor:
        osb = _check(x)
        B, L, C = x.shape
        H = attn.num_heads
        D, M4 = C // H, attn.linear2.in_features - C
        mod, _ = self._modulation(osb, attn.modulation, vec)
        x2 = x.reshape(B * L, C).contiguous()
        fp8 = getattr(vec, "_osb_fp8", None)
        if fp8 is not None and fp8.proj:
            return self._fp8_proj(osb, fp8, attn, x2, mod, B, L, C, H, D, pe, vec).view(B, L, C)
        xm = osb.ln_modulate(x2, mod.shift, mod.scale, group_rows=L)
        wq, bq, wm, bm = self._split_weights(attn)
        lo = self._split_lora(attn, M4)
        u = None if lo is None else osb.gemm(xm, lo[0][0])                       # shared down projection
        lq, lm = (None, None) if lo is None else lo
        qkv = _gemm(osb, xm, wq, bq, lq, u)                                      # [B*L, 3C]
        cos, sin, half = _rope(pe)
        kw = dict(q_norm_w=attn.norm.query_norm.scale, k_norm_w=attn.norm.key_norm.scale, rope_cos=cos, rope_sin=sin,
                  rope_half=half)
        if fp8 is not None:
            return self._fp8_tail(osb, fp8, attn, x2, qkv, mod, B, L, C, H, D, kw, vec).view(B, L, C)
        # [attn | gelu(mlp)] side by side: the attention output and the GELU GEMM write one [rows, C + 4C] buffer
        cat = _sp_attention(osb, qkv, C + M4, B, L, H, D, kw, 0, x.dtype, x.device, getattr(vec, "_osb_fp8_attn", None))
        _gemm(osb, xm, wm, bm, lm, u, epilogue=osb.EPI_BIAS_GELU_TANH, out=cat[:, C:])
        out = _gemm(osb, cat, *linear_parts(attn.linear2), epilogue=osb.EPI_BIAS_GATE_RES, residual=x2, gate=mod.gate,
                    group_rows=L)
        return out.view(B, L, C)

    @staticmethod
    def _fp8_proj(osb, fp8: Fp8State, attn: nn.Module, x2: Tensor, mod, B: int, L: int, C: int, H: int, D: int, pe,
                  vec: Tensor) -> Tensor:
        """x + gate * linear2(cat(attn, gelu(mlp))) with every Linear on FP8: ONE ln_modulate_fp8 pass feeds the qkv GEMM
        (bf16 q|k|v for the attention) and the mlp GEMM (GELU codes into columns C.. of the e4m3 cat buffer), the
        attention output fills columns 0..C-1 as e4m3 with its block scales, and linear2 is one block-scaled FP8 GEMM."""
        wq, sq, bq = fp8.proj_weights(osb, attn, "single")[:3]
        wm, sm, bm, w2, s2, b2 = fp8.weights(osb, attn, "single")
        rows, M4, dev, f8 = B * L, wm.shape[0], x2.device, torch.float8_e4m3fn
        lo = SingleStreamBlockProcessor._split_lora(attn, M4) if fp8.lora else None
        lq, lm = (None, None) if lo is None else lo
        l2 = fp8.mlp_lora(attn, "single")[1]
        x8, xs = osb.ln_modulate_fp8(x2, mod.shift, mod.scale, group_rows=L,
                                     out=fp8.buf("x8", rows, C, dtype=f8, device=dev), out_scale=fp8.buf("xs", rows, device=dev))
        u = fp8.down(osb, (id(attn), "linear1"), lq, x8, xs)   # one down projection for the qkv and mlp parts
        qkv = _gemm8(osb, x8, xs, wq, sq, bq, lq, u)
        cat8 = fp8.buf("cat8", rows, C + M4, dtype=f8, device=dev)
        cats = fp8.buf("cats", rows, (C + M4) // 128, device=dev)
        cos, sin, half = _rope(pe)
        kw = dict(q_norm_w=attn.norm.query_norm.scale, k_norm_w=attn.norm.key_norm.scale, rope_cos=cos, rope_sin=sin,
                  rope_half=half)
        _sp_attention(osb, qkv, C, B, L, H, D, kw, 0, x2.dtype, dev, getattr(vec, "_osb_fp8_attn", None),
                      out8=(cat8[:, :C], cats[:, :C // 128]))
        _gemm8(osb, x8, xs, wm, sm, bm, lm, u, epilogue=osb.EPI_BIAS_GELU_TANH_FP8, out=cat8[:, C:],
               out_scale=cats[:, C // 128:])
        return _gemm8(osb, cat8, cats, w2, s2, b2, l2, fp8.down(osb, (id(attn), "linear2"), l2, cat8, cats),
                      epilogue=osb.EPI_BIAS_GATE_RES, residual=x2, gate=mod.gate, group_rows=L)

    @staticmethod
    def _fp8_tail(osb, fp8: Fp8State, attn: nn.Module, x2: Tensor, qkv: Tensor, mod, B: int, L: int, C: int, H: int,
                  D: int, kw: dict, vec: Tensor) -> Tensor:
        """x + gate * linear2(cat(attn, gelu(mlp))) with the cat buffer in e4m3: the attention output is block-quantized
        into columns 0..C-1, the mlp part of linear1 (on its own FP8 LN+modulate) emits its GELU codes into columns C..,
        and linear2 is one block-scaled FP8 GEMM."""
        wm, sm, bm, w2, s2, b2 = fp8.weights(osb, attn, "single")
        l1, l2 = fp8.mlp_lora(attn, "single")
        rows, M4, dev, f8 = B * L, wm.shape[0], x2.device, torch.float8_e4m3fn
        cat8 = fp8.buf("cat8", rows, C + M4, dtype=f8, device=dev)
        cats = fp8.buf("cats", rows, (C + M4) // 128, device=dev)
        ao = _sp_attention(osb, qkv, C, B, L, H, D, kw, 0, x2.dtype, dev, getattr(vec, "_osb_fp8_attn", None))
        osb.quant_blocks_fp8(ao, out=cat8[:, :C], out_scale=cats[:, :C // 128])
        x8, xs = osb.ln_modulate_fp8(x2, mod.shift, mod.scale, group_rows=L,
                                     out=fp8.buf("x8", rows, C, dtype=f8, device=dev), out_scale=fp8.buf("xs", rows, device=dev))
        _gemm8(osb, x8, xs, wm, sm, bm, l1, fp8.down(osb, (id(attn), "single", "fc1"), l1, x8, xs),
               epilogue=osb.EPI_BIAS_GELU_TANH_FP8, out=cat8[:, C:], out_scale=cats[:, C // 128:])
        return _gemm8(osb, cat8, cats, w2, s2, b2, l2, fp8.down(osb, (id(attn), "linear2"), l2, cat8, cats),
                      epilogue=osb.EPI_BIAS_GATE_RES, residual=x2, gate=mod.gate, group_rows=L)


class SingleStreamBlock(nn.Module):
    def __init__(self, hidden_size: int, num_heads: int, mlp_ratio: float = 4.0, qk_scale: float | None = None,
                 fused_qkv: bool = True):
        super().__init__()
        self.hidden_dim = self.hidden_size = hidden_size
        self.num_heads, self.head_dim = num_heads, hidden_size // num_heads
        self.scale = qk_scale or self.head_dim**-0.5
        self.fused_qkv = fused_qkv
        self.mlp_hidden_dim = int(hidden_size * mlp_ratio)
        if fused_qkv:
            self.linear1 = nn.Linear(hidden_size, hidden_size * 3 + self.mlp_hidden_dim)
        else:
            self.q_proj = nn.Linear(hidden_size, hidden_size)
            self.k_proj = nn.Linear(hidden_size, hidden_size)
            self.v_mlp = nn.Linear(hidden_size, hidden_size + self.mlp_hidden_dim)
        self.linear2 = nn.Linear(hidden_size + self.mlp_hidden_dim, hidden_size)
        self.norm = QKNorm(self.head_dim)
        self.pre_norm = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.mlp_act = nn.GELU(approximate="tanh")
        self.modulation = Modulation(hidden_size, double=False)
        self.set_processor(SingleStreamBlockProcessor())

    def set_processor(self, processor) -> None:
        self.processor = processor

    def get_processor(self):
        return self.processor

    def forward(self, x: Tensor, vec: Tensor, pe, **kwargs) -> Tensor:
        return self.processor(self, x, vec, pe)


class LastLayer(nn.Module):
    """layers.py:391-402."""

    def __init__(self, hidden_size: int, patch_size: int, out_channels: int):
        super().__init__()
        self.norm_final = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.linear = nn.Linear(hidden_size, patch_size * patch_size * out_channels, bias=True)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 2 * hidden_size, bias=True))

    def forward(self, x: Tensor, vec: Tensor) -> Tensor:
        osb = _check(x)
        B, L, C = x.shape
        m = _linear(torch.nn.functional.silu(vec).contiguous(), self.adaLN_modulation[1]).float()
        shift, scale = m.chunk(2, dim=1)
        xm = osb.ln_modulate(x.reshape(B * L, C).contiguous(), shift, scale, group_rows=L)
        return _linear(xm, self.linear).view(B, L, -1)
